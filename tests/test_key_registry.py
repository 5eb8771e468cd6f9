"""Hidden signing keys in email app circuits (`"keyRegistryDepth": d` in a spec): the key's pubkeyHash stays private and
BinaryMerkleRoot proves it is a leaf of a Poseidon(2) Merkle registry, whose root is published instead.  CPU only: the
gadget against oracle/merkle.py, its soundness probe, the app circuit on the oracle witness with the key at the first,
a middle and the last leaf, the Poseidon records of the path (replayed by a Python permutation), the level counts with
and without the native Poseidon op, and every refusal.  tests/test_gpu_key_registry.py runs the GPU side."""
import ctypes

import pytest

import zkemail_b200 as z
from oracle import merkle
from r1cs_probe import probe
from test_app_commit import SALT, commit_spec, permutation_signals, poseidon_records, signed_commit_email
from zkutil import AssertFailed, oracle_check, oracle_witness

R = z.FR_MODULUS
DEPTH = 4
N_KEYS = 11                      # odd: the last leaf has no right sibling, its path reads zeros[0]
POSITIONS = [0, 5, N_KEYS - 1]


def registry_spec(style: int, depth: int = DEPTH) -> dict:
    return dict(commit_spec(style), keyRegistryDepth=depth)


def email_key_hash() -> int:
    return z.hash.poseidon_large(signed_commit_email().publicKey, 9, 242)


def oracle_registry(position: int, depth: int = DEPTH) -> z.KeyRegistry:
    """N_KEYS leaves, the email's key at `position`, the others arbitrary field elements; levels from the oracle."""
    leaves = [pow(7, 100 + i, R) for i in range(N_KEYS)]
    leaves[position] = email_key_hash()
    return z.KeyRegistry(depth, merkle.levels(leaves, depth))


def _tamper(w, var, value):
    bad = ctypes.create_string_buffer(w.buf.raw, len(w.buf))
    bad[32 * var:32 * var + 32] = (value % R).to_bytes(32, "little")
    w.buf, saved = bad, w.buf
    try:
        with pytest.raises(AssertFailed) as e:
            oracle_check(w.circuit, w)
    finally:
        w.buf = saved
    return str(e.value)


# ---- the gadget ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("depth", [1, 4, 20])
def test_binary_merkle_root_template(depth):
    c = z.Circuit("BinaryMerkleRoot", [depth])
    leaves = [pow(3, i + 1, R) for i in range(3 if depth > 1 else 2)]
    lv = merkle.levels(leaves, depth)
    for i in range(len(leaves)):
        sib = merkle.path(lv, i)
        w = oracle_witness(c, {"leaf": leaves[i], "index": i, "siblings": sib})      # checks every row
        assert w.values("root") == [lv[-1][0]]
        assert merkle.check_path(lv[-1][0], leaves[i], i, sib)
    assert len(poseidon_records(c)) == depth and all(b["t"] == 3 for b in poseidon_records(c))


def test_tampered_path_fails_in_gadget():
    depth = 4
    c = z.Circuit("BinaryMerkleRoot", [depth])
    lv = merkle.levels([11, 12, 13, 14, 15], depth)
    w = oracle_witness(c, {"leaf": 13, "index": 2, "siblings": merkle.path(lv, 2)})
    first = c.groups["siblings"][0]
    assert _tamper(w, first + 1, w[first + 1] + 1).endswith("in BinaryMerkleRoot")
    # the index bits: variables right after the inputs (Num2Bits inside the gadget); bit 1 of index 2 flipped to 0
    bit1 = c.groups["siblings"][0] + depth + 1
    assert w[bit1] == 1
    assert _tamper(w, bit1, 0).endswith("in Num2Bits")
    with pytest.raises(AssertFailed, match="in Num2Bits"):
        oracle_witness(c, {"leaf": 13, "index": 1 << depth, "siblings": merkle.path(lv, 2)})
    with pytest.raises(z._lib.ZkeError, match="depth must be 1..32"):
        z.Circuit("BinaryMerkleRoot", [33])


def test_gadget_has_no_free_variable():
    depth = 5
    c = z.Circuit("BinaryMerkleRoot", [depth])
    lv = merkle.levels(list(range(1, 20)), depth)
    w = oracle_witness(c, {"leaf": 6, "index": 5, "siblings": merkle.path(lv, 5)})
    free, two, unmentioned = probe(c, [w[i] for i in range(c.info.n_vars)])
    assert not free and not two and not unmentioned, (free, two, unmentioned)


# ---- the app circuit -------------------------------------------------------------------------------------------------

_APPS = {}


def _app(style):
    if style not in _APPS:
        spec = registry_spec(style)
        _APPS[style] = (spec, z.Circuit.from_spec(spec))
    return _APPS[style]


def _inputs(spec, reg):
    return z.generate_app_inputs(signed_commit_email(), spec, {"senderSalt": SALT, "recipient": 77}, params={"registry": reg})


@pytest.mark.parametrize("position", POSITIONS, ids=["first", "middle", "last"])
@pytest.mark.parametrize("style", [0, 1], ids=["zkregex", "compact"])
def test_app_registry_root(style, position):
    spec, c = _app(style)
    reg = oracle_registry(position)
    inputs = _inputs(spec, reg)
    assert inputs["registryIndex"] == str(position)
    w = oracle_witness(c, inputs)                                   # checks every constraint
    outs = [g for g, (_, _, kind) in c.groups.items() if kind == 0]
    assert outs == ["registryRoot", "shaHi", "shaLo", "sender", "order", "note"] and "pubkeyHash" not in c.groups
    assert list(c.groups)[-2:] == ["registryIndex", "registrySiblings"]
    assert c.groups["registrySiblings"][1] == DEPTH
    out = z.decode_app_outputs(spec, [w[1 + i] for i in range(c.info.n_public)])
    assert "pubkeyHash" not in out
    assert out["registryRoot"] == merkle.root(reg.leaves, DEPTH) == reg.root
    assert merkle.check_path(reg.root, email_key_hash(), position, [int(x) for x in inputs["registrySiblings"]])


def test_app_records_match_oracle():
    spec, c = _app(1)
    w = oracle_witness(c, _inputs(spec, oracle_registry(5)))
    blocks = poseidon_records(c)
    assert [b["t"] for b in blocks] == [3] * DEPTH + [4, 3, 2, 17, 5, 3]    # the path first (it precedes the app's scope)
    for b in blocks:
        vals = permutation_signals(b["t"], [0] + [w[v] for v in b["inputs"]])
        seen = set()
        for k in range(0, len(b["desc"]), 2):
            var, word = b["desc"][k], b["desc"][k + 1]
            assert w[var] == vals[(word >> 16, (word >> 8) & 0xff, word & 0xff)]
            seen.add(var)
        assert seen == set(range(*b["var"]))
    assert w[blocks[DEPTH - 1]["desc"][-2]] == w[c.groups["registryRoot"][0]]


def test_native_poseidon_levels():
    spec, c = _app(1)
    plain = z.Circuit.from_spec(commit_spec(1))
    for cl in (1, 8):
        on, off = c.program_stats(cluster=cl), c.program_stats(cluster=cl, native_poseidon=False)
        assert on["n_levels"] < off["n_levels"]
        assert off["n_coop_ops"] - on["n_coop_ops"] == -(6 + DEPTH)
        # per tree level: the swap product, left / right, one native Poseidon op
        assert on["n_levels"] <= plain.program_stats(cluster=cl)["n_levels"] + 3 * DEPTH


def test_depth_zero_is_todays_circuit():
    for style in (0, 1):
        a, b = z.Circuit.from_spec(commit_spec(style)), z.Circuit.from_spec(registry_spec(style, 0))
        assert a.write_r1cs() == b.write_r1cs() and a.groups == b.groups
        for cl in (1, 8):
            assert a.program_stats(cluster=cl)["digest"] == b.program_stats(cluster=cl)["digest"]


def _refused(spec, *needles):
    with pytest.raises(z._lib.ZkeError) as e:
        z.Circuit.from_spec(spec)
    for n in needles:
        assert n in str(e.value), str(e.value)


def test_refusals():
    base = {"maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": 1, "keyRegistryDepth": 3}
    _refused(dict(base, keyRegistryDepth=33), "keyRegistryDepth", "at most 32")
    _refused(dict(base, keyRegistryDepth=2.5), "keyRegistryDepth", "integer")
    _refused(dict(base, keyRegistryDepth="4"), "keyRegistryDepth", "integer")
    _refused(dict(base, keyRegistryDepth=-1), "keyRegistryDepth", "integer")
    _refused(dict(base, publicPubkey=True), "keyRegistryDepth", "publicPubkey")

    def rx(name):
        return [{"name": name, "location": "header",
                 "parts": [{"regexDef": "(\r\n|^)subject:"}, {"regexDef": "[^\r\n]+", "isPublic": True, "maxLength": 32}]}]
    _refused(dict(base, regexes=rx("registryRoot")), "regexes[0].name", "'registryRoot'", "key registry")
    _refused(dict(base, regexes=rx("registry")), "regexes[0].name", "'registryIndex'", "key registry")
    _refused(dict(base, externalInputs=[{"name": "registrySiblings"}]), "externalInputs[0].name", "'registrySiblings'")
    off = dict(base, keyRegistryDepth=0)
    for spec in (dict(off, regexes=rx("registryRoot")), dict(off, regexes=rx("registry")),
                 dict(off, externalInputs=[{"name": "registrySiblings", "isPublic": False}])):
        z.Circuit.from_spec(spec)                                   # the names are free without a registry
    assert "registryRoot" in z.Circuit.from_spec(dict(off, regexes=rx("registryRoot"))).groups


def test_input_refusals():
    spec = registry_spec(1)
    with pytest.raises(ValueError, match="registry"):
        z.generate_app_inputs(signed_commit_email(), spec, {"senderSalt": SALT, "recipient": 77})
    leaves = [pow(7, 100 + i, R) for i in range(N_KEYS)]
    with pytest.raises(ValueError, match="depth"):
        _inputs(spec, z.KeyRegistry(DEPTH + 1, merkle.levels(leaves, DEPTH + 1)))
    with pytest.raises(ValueError, match="not in the registry"):
        _inputs(spec, z.KeyRegistry(DEPTH, merkle.levels(leaves, DEPTH)))
    with pytest.raises(ValueError, match="level 1"):
        z.KeyRegistry(2, [[1, 2, 3], [4], [5]])
    with pytest.raises(ValueError, match="depth"):
        z.KeyRegistry(0, [[1]])


def test_registry_host_side():
    reg = oracle_registry(5)
    i, sib = reg.path(5)
    assert i == 5 and sib == merkle.path(reg.levels, 5)
    assert reg.path(N_KEYS - 1)[1][0] == 0                          # zeros[0]
    assert reg.zeros() == merkle.zeros(DEPTH)
    assert reg.index_of(email_key_hash()) == 5
    assert '"depth": 4' in reg.to_json()


def test_native_calls_refuse_bad_arguments():
    """Argument checks come before the device: these refusals hold with or without a GPU."""
    L = z._lib
    err = ctypes.create_string_buffer(L.ERRCAP)
    out = ctypes.create_string_buffer(64)
    assert L.zke_poseidon_batch(bytes(32 * 17), 17, 1, 0, out, err, L.ERRCAP) < 0 and b"width" in err.value
    assert L.zke_poseidon_batch(bytes(32), 0, 1, 0, out, err, L.ERRCAP) < 0 and b"width" in err.value
    assert L.zke_pubkey_hashes(bytes(256), 1, 256, 121, 16, 0, out, err, L.ERRCAP) < 0 and b"k must be 17..32" in err.value
    assert L.zke_pubkey_hashes(bytes(256), 1, 256, 126, 17, 0, out, err, L.ERRCAP) < 0 and b"2n < 251" in err.value
    assert L.zke_merkle_build(bytes(32), 0, 4, 0, None, 0, err, L.ERRCAP) < 0 and b"count" in err.value
    assert L.zke_merkle_build(bytes(32 * 3), 3, 1, 0, None, 0, err, L.ERRCAP) < 0 and b"does not fit" in err.value
    assert L.zke_merkle_build(bytes(32), 1, 0, 0, None, 0, err, L.ERRCAP) < 0 and b"depth must be 1..32" in err.value
    assert L.zke_merkle_build(bytes(32), 1, 33, 0, None, 0, err, L.ERRCAP) < 0 and b"depth must be 1..32" in err.value
    assert L.zke_merkle_build(bytes(32 * 3), 3, 2, 0, None, 0, err, L.ERRCAP) == 32 * (3 + 2 + 1)
    assert L.zke_merkle_build(bytes(32 * 3), 3, 2, 0, out, 64, err, L.ERRCAP) == -2
    if z.device_count() == 0:
        assert L.zke_poseidon_batch(bytes(32), 1, 1, 0, out, err, L.ERRCAP) < 0 and b"no CPU fallback" in err.value
