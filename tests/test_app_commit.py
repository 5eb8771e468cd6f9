"""Hashed and committed reveals of email app circuits (`"reveal": "hash" | "commit"` in a spec): the part's packed bytes
go through PoseidonModular (utils/hash.circom), optionally followed by Poseidon(2) with a private salt, and only that hash
is public.  CPU only: the host Poseidon (zke_poseidon_hash, zkemail_b200.hash) against the oracle and a restatement of the
helpers' hash.ts, the circuits' outputs on the oracle witness, the refusals, the Poseidon record the engine's native op
reads (checked by a Python permutation over the oracle witness), and the level counts of the lowering with and without
that op.  tests/test_gpu_app_commit.py runs the device op."""
import copy
import ctypes
import random

import pytest

import zkemail_b200 as z
from oracle import poseidon as oracle_poseidon
from zkutil import AssertFailed, oracle_check, oracle_witness

R = z.FR_MODULUS

SALT = 0x1234_5678_9abc_def0_0fed_cba9_8765_4321
LONG_NOTE = ("the quick brown fox jumps over the lazy dog " * 14)[:600]    # > 496 bytes: two chunk hashes


def commit_spec(style: int) -> dict:
    """EmailVerifier(640, 768) with a committed sender address (the hidden-sender pattern), a hashed order id and a
    hashed long note (20 packed words: Poseidon(16), Poseidon(4), then Poseidon(2) to chain them), one public and one
    private external input."""
    return {
        "maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": style,
        "regexes": [
            {"name": "sender", "location": "header",
             "parts": [{"regexDef": "(\r\n|^)from:"}, {"regexDef": "([^\r\n]+<)?"},
                       {"regexDef": "[a-zA-Z0-9._%+-]+@[a-zA-Z0-9.-]+", "isPublic": True, "maxLength": 64,
                        "reveal": "commit", "salt": "senderSalt"},
                       {"regexDef": ">?\r\n"}]},
            {"name": "order", "location": "body",
             "parts": [{"regexDef": "Order #"}, {"regexDef": "[0-9]+", "isPublic": True, "maxLength": 5, "reveal": "hash"}]},
            {"name": "note", "location": "body",
             "parts": [{"regexDef": "Note: "}, {"regexDef": "[a-z ]+", "isPublic": True, "maxLength": 620, "reveal": "hash"},
                       {"regexDef": "\r\n"}]},
        ],
        "externalInputs": [{"name": "senderSalt", "isPublic": False}, {"name": "recipient"}],
    }


def commit_body(order: str, note: str) -> bytes:
    return b"Dear customer,\r\nOrder #" + order.encode() + b" has shipped.\r\nNote: " + note.encode() + b"\r\nThanks\r\n"


def signed_commit_email(index: int = 3, order: str = "40213", note: str = LONG_NOTE):
    key = z.synthetic.generate_key(seed=77)
    em = z.synthetic.make_signed_email(index, key, domain="gmail.com", body_override=commit_body(order, note))
    return z.verify_dkim_signature(em, resolver=lambda n, t: [z.synthetic.key_record(key)])


def sender_of(index: int) -> str:
    return f"sender{index:04d}@gmail.com"


# ---- host Poseidon ---------------------------------------------------------------------------------------------------

def test_host_poseidon_all_widths():
    rng = random.Random(11)
    for n in range(1, 17):                                          # widths 2..17
        xs = [rng.randrange(R) for _ in range(n)]
        xs[0] = R - 1
        want = oracle_poseidon.poseidon(xs)
        assert z.hash.poseidon(xs) == want
        out = ctypes.create_string_buffer(32)
        assert z._lib.zke_poseidon_hash(b"".join(x.to_bytes(32, "little") for x in xs), n, out) == 0
        assert int.from_bytes(out.raw, "little") == want
    assert z.hash.poseidon([1, 2]) == 0x115cc0f5e7d690413df64c6b9662e9cf2a3617f2743245519e19607a4417189a   # circomlib vector
    assert z.hash.poseidon([R + 5]) == z.hash.poseidon([5])         # reduced mod r, as circomlibjs does
    out = ctypes.create_string_buffer(32)
    assert z._lib.zke_poseidon_hash(R.to_bytes(32, "little"), 1, out) == -2
    assert z._lib.zke_poseidon_hash(bytes(32 * 17), 17, out) == -1
    assert z._lib.zke_poseidon_hash(bytes(32), 0, out) == -1
    with pytest.raises(ValueError):
        z.hash.poseidon(list(range(17)))


def hash_ts_poseidon_modular(inputs):
    """packages/helpers/src/hash.ts: poseidonModular, restated line by line on the oracle's permutation."""
    CHUNK_SIZE = 16
    num_elements = len(inputs)
    chunks = num_elements // CHUNK_SIZE
    last_chunk_size = num_elements % CHUNK_SIZE
    if last_chunk_size != 0:
        chunks += 1
    out = None
    for i in range(chunks):
        start = i * CHUNK_SIZE
        end = start + CHUNK_SIZE
        if end > num_elements:
            end = num_elements
        chunk_hash = oracle_poseidon.poseidon(inputs[start:end])
        out = chunk_hash if i == 0 else oracle_poseidon.poseidon([out, chunk_hash])
    if out is None:
        raise ValueError("No inputs provided")
    return out


@pytest.mark.parametrize("n", [1, 16, 17, 33, 48])
def test_poseidon_modular_matches_hash_ts(n):
    rng = random.Random(n)
    xs = [rng.randrange(R) for _ in range(n)]
    assert z.hash.poseidon_modular(xs) == hash_ts_poseidon_modular(xs) == oracle_poseidon.poseidon_modular(xs)


def test_poseidon_large_and_empty_input():
    v = random.Random(3).getrandbits(2048)
    assert z.hash.poseidon_large(v, 9, 242) == oracle_poseidon.poseidon_large(v, 9, 242)
    with pytest.raises(ValueError, match="No inputs provided"):
        z.hash.poseidon_modular([])


# ---- circuits --------------------------------------------------------------------------------------------------------

def _same_circuit(a, b):
    assert a.write_r1cs() == b.write_r1cs()
    assert a.groups == b.groups
    for cl in (1, 8):
        assert a.program_stats(cluster=cl)["digest"] == b.program_stats(cluster=cl)["digest"]


def test_default_keys_change_nothing():
    """"reveal": "bytes" and "isPublic": true are today's circuit, byte for byte, with no Poseidon record."""
    from test_app_circuit import app_spec
    spec = app_spec(1)
    explicit = copy.deepcopy(spec)
    for rx in explicit["regexes"]:
        for p in rx["parts"]:
            if p.get("isPublic"):
                p["reveal"] = "bytes"
    for ei in explicit["externalInputs"]:
        ei["isPublic"] = True
    a, b = z.Circuit.from_spec(spec), z.Circuit.from_spec(explicit)
    _same_circuit(a, b)
    assert poseidon_records(a) == []
    assert a.program_stats(native_poseidon=False)["digest"] == a.program_stats()["digest"]


@pytest.fixture(scope="module", params=[0, 1], ids=["zkregex", "compact"])
def app(request):
    spec = commit_spec(request.param)
    c = z.Circuit.from_spec(spec)
    inputs = z.generate_app_inputs(signed_commit_email(), spec, {"senderSalt": SALT, "recipient": 77})
    return spec, c, inputs, oracle_witness(c, inputs)               # checks every constraint


def test_signal_layout(app):
    spec, c, inputs, _ = app
    kinds = {g: kind for g, (_, _, kind) in c.groups.items()}
    assert [g for g, k in kinds.items() if k == 0] == ["pubkeyHash", "shaHi", "shaLo", "sender", "order", "note"]
    assert [g for g, k in kinds.items() if k == 1] == ["recipient"]
    assert list(c.groups)[-4:] == ["senderIndex", "orderIndex", "noteIndex", "senderSalt"]    # the salt comes last
    assert all(c.groups[n][1] == 1 for n in ("sender", "order", "note", "senderSalt"))
    assert c.info.n_public == 7


def test_outputs(app):
    spec, c, inputs, w = app
    out = z.decode_app_outputs(spec, [w[1 + i] for i in range(c.info.n_public)])
    assert set(out) == {"pubkeyHash", "shaHi", "shaLo", "sender", "order", "note", "recipient"}
    pk = lambda s, n: [int(x) for x in z.app.pack_bytes(s.encode(), n)]
    h_sender = z.hash.poseidon_modular(pk(sender_of(3), 64))
    assert out["order"] == z.hash.poseidon_modular(pk("40213", 5)) == oracle_poseidon.poseidon_modular(pk("40213", 5))
    assert out["note"] == z.hash.poseidon_modular(pk(LONG_NOTE, 620))
    assert out["sender"] == z.hash.poseidon([h_sender, SALT]) == oracle_poseidon.poseidon([h_sender, SALT])
    assert out["recipient"] == 77
    for name, value, salt in (("sender", sender_of(3), SALT), ("order", "40213", None), ("note", LONG_NOTE, None)):
        assert z.expected_app_output(spec, name, value, salt) == out[name]
    assert z.expected_app_output(spec, "sender", sender_of(3), SALT + 1) != out["sender"]
    with pytest.raises(ValueError, match="salt"):
        z.expected_app_output(spec, "sender", sender_of(3))


def test_other_salt_other_commitment(app):
    spec, c, inputs, w = app
    w2 = oracle_witness(c, dict(inputs, senderSalt=str(R - 1)))
    first = c.groups["sender"][0]
    assert w2[first] != w[first]
    assert w2[first] == z.expected_app_output(spec, "sender", sender_of(3), R - 1)
    assert w2.values("order") == w.values("order")


def test_tampered_poseidon_signal_fails_in_poseidon(app):
    _, c, _, w = app
    blk = poseidon_records(c)[0]
    var = blk["desc"][2 * (len(blk["desc"]) // 4)]                   # a signal half way through the permutation
    bad = ctypes.create_string_buffer(w.buf.raw, len(w.buf))
    bad[32 * var:32 * var + 32] = ((w[var] + 1) % R).to_bytes(32, "little")
    w.buf, saved = bad, w.buf
    try:
        with pytest.raises(AssertFailed, match="in Poseidon$"):
            oracle_check(c, w)
    finally:
        w.buf = saved


def test_shifted_index_fails(app):
    _, c, inputs, _ = app
    for name in ("senderIndex", "orderIndex", "noteIndex"):
        with pytest.raises(AssertFailed):
            oracle_witness(c, dict(inputs, **{name: str(int(inputs[name]) + 1)}))


def _refused(spec, *needles):
    with pytest.raises(z._lib.ZkeError) as e:
        z.Circuit.from_spec(spec)
    for n in needles:
        assert n in str(e.value), str(e.value)


def test_refusals():
    base = {"maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": 1}
    salt = {"name": "s", "isPublic": False}

    def spec(part, externals=(salt,)):
        return dict(base, regexes=[{"name": "a", "location": "header",
                                    "parts": [{"regexDef": "(\r\n|^)subject:"}, part]}], externalInputs=list(externals))
    pub = {"regexDef": "[^\r\n]+", "isPublic": True, "maxLength": 32}
    _refused(spec({"regexDef": "[^\r\n]+", "reveal": "hash"}), "regexes[0].parts[1].reveal", "only a public part")
    _refused(spec(dict(pub, reveal="sha")), "regexes[0].parts[1].reveal", "'sha'")
    _refused(spec(dict(pub, reveal=1)), "regexes[0].parts[1].reveal", "expected a string")
    _refused(spec(dict(pub, reveal="hash", salt="s")), "regexes[0].parts[1].salt", "needs reveal \"commit\"")
    _refused(spec(dict(pub, salt="s")), "regexes[0].parts[1].salt", "needs reveal \"commit\"")
    _refused(spec({"regexDef": "[^\r\n]+", "salt": "s"}), "regexes[0].parts[1].salt", "only a public part")
    _refused(spec(dict(pub, reveal="commit")), "regexes[0].parts[1].salt", "needs a salt")
    _refused(spec(dict(pub, reveal="commit", salt="t")), "regexes[0].parts[1].salt", "no external input named 't'")
    _refused(spec(dict(pub, reveal="commit", salt="s"), [{"name": "s"}]), "regexes[0].parts[1].salt", "is public")
    _refused(spec(dict(pub, reveal="commit", salt="s"), [{"name": "s", "isPublic": False, "maxLength": 31}]),
             "regexes[0].parts[1].salt", "is packed")
    _refused(spec(dict(pub, reveal="hash", maxLength=641)), "regexes[0].parts[1].maxLength", "larger than the searched header")
    _refused(spec(dict(pub, reveal="hash"), [{"name": "s", "isPublic": "no"}]), "externalInputs[0].isPublic", "true or false")
    c = z.Circuit.from_spec(spec(dict(pub, reveal="commit", salt="s")))
    assert c.info.n_public == 4 and c.groups["s"][2] == 2


# ---- the Poseidon record (ZKE_ARR_POSEIDON_BLOCKS) -------------------------------------------------------------------

def poseidon_records(c):
    L = z._lib
    n = L.c_size_t()
    p = L.zke_circuit_array(c.handle, L.ARR_POSEIDON_BLOCKS, ctypes.byref(n))
    flat = list((ctypes.c_uint32 * n.value).from_address(p)) if n.value else [0]
    out, pos = [], 1
    for _ in range(flat[0]):
        t, vb, ve, tb, te, nd = flat[pos:pos + 6]
        pos += 6
        inputs = flat[pos:pos + t - 1]; pos += t - 1
        desc = flat[pos:pos + 2 * nd]; pos += 2 * nd
        out.append({"t": t, "var": (vb, ve), "temp": (tb, te), "inputs": inputs, "desc": desc})
    assert pos == len(flat)
    return out


def permutation_signals(t, state):
    """{(round, lane, kind): value} of the plain permutation (kinds of circuit.hpp: PoseidonKind)."""
    rc, mds = oracle_poseidon.params(t)
    r_p = oracle_poseidon.N_ROUNDS_P[t - 2]
    vals = {(0, i, 0): state[i] for i in range(1, t)}
    st = list(state)
    for rnd in range(8 + r_p):
        st = [(s + rc[rnd * t + i]) % R for i, s in enumerate(st)]
        for i in range(t if rnd < 4 or rnd >= 4 + r_p else 1):
            x2 = st[i] * st[i] % R
            x4 = x2 * x2 % R
            st[i] = x4 * st[i] % R
            vals[(rnd, i, 1)], vals[(rnd, i, 2)], vals[(rnd, i, 3)] = x2, x4, st[i]
        st = [sum(mds[i][j] * st[j] for j in range(t)) % R for i in range(t)]
        for i in range(t):
            vals[(rnd, i, 4)] = st[i]
    return vals


def test_record_matches_oracle(app):
    spec, c, inputs, w = app
    blocks = poseidon_records(c)
    # sender: Poseidon(3) then the commitment Poseidon(2); order: Poseidon(1); note: Poseidon(16), Poseidon(4), Poseidon(2)
    assert [b["t"] for b in blocks] == [4, 3, 2, 17, 5, 3]
    for b in blocks:
        vals = permutation_signals(b["t"], [0] + [w[v] for v in b["inputs"]])
        seen = set()
        for k in range(0, len(b["desc"]), 2):
            var, word = b["desc"][k], b["desc"][k + 1]
            key = (word >> 16, (word >> 8) & 0xff, word & 0xff)
            assert w[var] == vals[key], (b["t"], key)
            seen.add(var)
        assert seen == set(range(*b["var"]))                          # every created signal exactly once
        # mix sums of more than 8 terms (t >= 8) are split into three scratch partial sums each (circuit.cpp: LC_FANIN)
        n_mix = (8 + oracle_poseidon.N_ROUNDS_P[b["t"] - 2]) * b["t"] - (b["t"] - 1)
        assert b["temp"][1] - b["temp"][0] == (0 if b["t"] <= 7 else 3 * n_mix)
    salt_var = c.groups["senderSalt"][0]
    assert blocks[1]["inputs"] == [blocks[0]["desc"][-2], salt_var]   # the commitment hashes the chunk hash and the salt
    assert w[salt_var] == SALT


def test_native_poseidon_levels(app):
    """The native op replaces each recorded instance's ~4 levels per round by one level.  The hash chain of a revealed
    part starts after its regex and PackRegexReveal, so the serial Poseidons of the longest chain (sender: two, note: two
    after the parallel chunk hashes) add their levels to the program's depth without the op."""
    spec, c, _, _ = app
    plain = copy.deepcopy(spec)
    for rx in plain["regexes"]:
        for p in rx["parts"]:
            p.pop("reveal", None)
            p.pop("salt", None)
    depth_plain = z.Circuit.from_spec(plain).program_stats()["n_levels"]
    for cl in (1, 8):
        on, off = c.program_stats(cluster=cl), c.program_stats(cluster=cl, native_poseidon=False)
        assert off["n_coop_ops"] - on["n_coop_ops"] == -6
        assert off["n_levels"] - on["n_levels"] >= 250            # 342 -> 683 levels at EmailVerifier(640, 768)
        assert on["n_levels"] <= depth_plain + 2                   # the hashes add (almost) no depth over plain reveals
        assert on["n_ops_kept"] < off["n_ops_kept"]
