"""Domain-bound registry leaves on the GPU: zke_domain_key_leaves against the oracle leaf (edge rows, counts around the
block size, k = 17 where the key and domain hashes share their constants and k = 32 where three sets are staged), each
refusal naming its row, then an app with `"keyDomain"` on the DKIM `d=` tag: its GPU witness against the CPU oracle bit
for bit (cluster widths default, 1 and 8, native Poseidon on and off), its proof at fixed (r, s) against the oracle's
under every verifier, and 64 emails over four (domain, key) pairs - one key under two domains, one domain with two
keys - proved in one batch, each publishing the registry's root and its own domain."""
import ctypes
import functools
import random

import pytest

import zkemail_b200 as z
import zkutil
from oracle import merkle
from test_app_commit import SALT, commit_body
from test_domain_registry import domain_spec, oracle_domain_key_leaf
from zkutil import oracle_witness

pytestmark = pytest.mark.gpu

R = z.FR_MODULUS
L = z._lib
DEPTH = 10


def _rows(domains):
    return b"".join(d.ljust(255, b"\0") for d in domains)


def _leaves_raw(moduli, domains, n=121, k=17):
    mbytes = (n * k + 7) // 8
    out, err = ctypes.create_string_buffer(32 * len(moduli)), ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_domain_key_leaves(b"".join(m.to_bytes(mbytes, "little") for m in moduli), len(moduli), mbytes, n, k,
                                 _rows(domains), 0, out, err, L.ERRCAP)
    return rc, err.value.decode(), [int.from_bytes(out.raw[32 * i:32 * i + 32], "little") for i in range(len(moduli))]


def _pairs(count, seed, n=121, k=17):
    rng = random.Random(seed)
    moduli = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(count)]
    alphabet = b"abcdefghijklmnopqrstuvwxyz0123456789-."
    domains = []
    for _ in range(count):
        length = rng.randrange(1, 64)
        d = bytes(rng.choice(alphabet[:36]) if j in (0, length - 1) else rng.choice(alphabet) for j in range(length))
        domains.append(d)
    edges = [(b"a", (1 << (n * k)) - 1), (b"x" * 255, moduli[0]), (b"b" * 31, 3), (b"c" * 32, 1 << 2047),
             (b"d" * 62, (1 << (n * k)) - 1), (b"xn--bcher-kva.example", moduli[-1])]
    for i, (d, m) in enumerate(edges[:count]):
        domains[i], moduli[i] = d, m
    return moduli, domains


def test_leaves_match_oracle_1000_pairs():
    moduli, domains = _pairs(1000, 1)
    rc, err, got = _leaves_raw(moduli, domains)
    assert rc == 0, err
    assert got == [oracle_domain_key_leaf(d, m) for d, m in zip(domains, moduli)]
    assert z.registry.domain_key_leaves([(d.decode(), m) for d, m in zip(domains, moduli)]) == got


@pytest.mark.parametrize("count", [1, 127, 128, 129, 65537])
def test_leaves_at_counts(count):
    """Every leaf against the host leaf (zke_poseidon_hash); against the oracle every leaf up to 129 and every 61st
    (plus the ends) at 65,537."""
    moduli, domains = _pairs(count, count)
    rc, err, got = _leaves_raw(moduli, domains)
    assert rc == 0, err
    check = range(count) if count <= 129 else sorted(set(range(0, count, 61)) | {count - 2, count - 1})
    for i in check:
        assert got[i] == oracle_domain_key_leaf(domains[i], moduli[i]), i
    host = range(count) if count <= 129 else range(0, count, 7)
    for i in host:
        assert got[i] == z.registry.domain_key_leaf(domains[i].decode(), moduli[i]), i
    assert L.zke_registry_device_ms() > 0


@pytest.mark.parametrize("k", [17, 32])
def test_leaves_at_key_widths(k):
    """k = 17: the key's Poseidon(9) shares the domain's constants (two sets staged); k = 32: Poseidon(16), three sets
    and more than the default 48 KB of shared memory."""
    n = 121
    moduli, domains = _pairs(300, k, n, k)
    moduli[1] = (1 << (n * k)) - 1
    rc, err, got = _leaves_raw(moduli, domains, n, k)
    assert rc == 0, err
    assert got == [oracle_domain_key_leaf(d, m, n, k) for d, m in zip(domains, moduli)]


def test_refusals_name_the_row():
    moduli, domains = _pairs(200, 3)
    for row, bad, needle in ((37, b"Gmail.com", "upper-case byte at 0"), (5, b"gmail\0com", "zero byte at 5"),
                             (150, b"", "is empty"), (199, b"gmail.com.", "ends with a dot"),
                             (64, b"b\xc3\xbccher.de", "non-ASCII byte at 1")):
        ds = list(domains)
        ds[row] = bad
        if row < 190:
            ds[190] = b"Late.example"                              # a later bad row: the first one is named
        rc, err, _ = _leaves_raw(moduli, ds)
        assert rc < 0 and f"domain {row} is not canonical" in err and needle in err, err
    ms = list(moduli)
    ms[77] = 1 << (121 * 17)
    rc, err, _ = _leaves_raw(ms, domains)
    assert rc < 0 and "modulus 77 is not below 2^(n k)" in err, err


# ---- the app -----------------------------------------------------------------------------------------------------------

_key = functools.lru_cache(maxsize=None)(lambda seed: z.synthetic.generate_key(seed=seed))

# one key under two domains (77), one domain with two keys (78 and 79: a rotation)
SIGNERS = [("corp77.com", 77), ("alias77.org", 77), ("corp78.com", 78), ("corp78.com", 79)]
SLOTS = [0, 333, 998, 999]


def _signed(i, domain, seed):
    key = _key(seed)
    em = z.synthetic.make_signed_email(i, key, domain=domain, body_override=commit_body(str(1000 + i), "a note"))
    return z.verify_dkim_signature(em, resolver=lambda n, t: [z.synthetic.key_record(key)])


_APP = {}


def _app():
    if not _APP:
        spec = domain_spec(1, "dkim", depth=DEPTH)
        c = z.Circuit.from_spec(spec)
        rng = random.Random(9)
        pairs = [(f"filler{i}.example", rng.getrandbits(2048) | (1 << 2047) | 1) for i in range(1000)]
        for slot, (domain, seed) in zip(SLOTS, SIGNERS):
            pairs[slot] = (domain.upper() + ".", z.synthetic.key_record(_key(seed)))   # canonicalised by build_domains
        reg = z.KeyRegistry.build_domains(pairs, DEPTH)
        assert reg.domain_bound and reg.root == merkle.root(reg.leaves, DEPTH)
        for slot, (domain, seed) in zip(SLOTS, SIGNERS):
            assert reg.leaves[slot] == oracle_domain_key_leaf(domain.encode(), _key(seed).public_key().public_numbers().n)
        back = z.KeyRegistry.from_json(reg.to_json())
        assert back.levels == reg.levels and back.domain_bound
        dks = [_signed(slot, domain, seed) for slot, (domain, seed) in zip(SLOTS, SIGNERS)]
        inputs = [z.generate_app_inputs(dk, spec, {"senderSalt": SALT + j, "recipient": j}, params={"registry": reg})
                  for j, dk in enumerate(dks)]
        assert [x["registryIndex"] for x in inputs] == [str(s) for s in SLOTS]
        _APP.update(spec=spec, c=c, reg=reg, inputs=inputs, refs=[oracle_witness(c, x).raw() for x in inputs])
    return _APP


@pytest.mark.parametrize("native", ["1", "0"], ids=["native", "gadget"])
@pytest.mark.parametrize("width", ["default", "1", "8"])
def test_domain_witness_matches_oracle(width, native, monkeypatch):
    if width == "default":
        monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    monkeypatch.setenv("ZKE_NATIVE_POSEIDON", native)
    a = _app()
    c, order = a["c"], [0, 1, 2, 3, 3, 0]
    ctx = z.Context(c, None, device=0, max_batch=len(order))
    wt, status = ctx.witness(b"".join(c.pack_inputs(a["inputs"][e]) for e in order), len(order))
    m = 32 * c.info.n_vars
    assert status == [-1] * len(order)
    for k, e in enumerate(order):
        assert wt[k * m:(k + 1) * m] == a["refs"][e], f"email {k} (input {e}) differs from the oracle"


def test_domain_proofs(monkeypatch):
    from oracle import bn254
    monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    monkeypatch.delenv("ZKE_NATIVE_POSEIDON", raising=False)
    a = _app()
    c, spec, reg = a["c"], a["spec"], a["reg"]
    zk = z.Zkey(c, seed=29)
    vk = zk.vkey()

    ctx = z.Context(c, zk, device=0, max_batch=1)
    wt, status = ctx.witness(c.pack_inputs(a["inputs"][2]), 1)
    assert status == [-1] and wt == a["refs"][2]
    r, s = 717171, 828282
    proofs, publics, _ = ctx.prove(1, r.to_bytes(32, "little") + s.to_bytes(32, "little"))
    assert proofs == zkutil.oracle_prove(c, zkutil.product_sections(zk), wt, r, s)
    proof, pubs = z.proof_to_json(proofs, publics, c.info.n_public)
    assert bn254.groth16_verify(vk, pubs, proof) and z.verify(vk, pubs, proof)
    assert z.Verifier(vk, device=0).verify_batch([pubs], [proof]) == [True]
    assert z.verify_batch(vk, [pubs], [proof]) == [True]
    out = z.decode_app_outputs(spec, pubs)
    assert out["registryRoot"] == reg.root and out["dkimDomain"] == "corp78.com"
    del ctx

    # 64 emails, 16 per (domain, key) pair, one proving key: every proof publishes the root and its own domain
    batch = 64
    inputs, want = [], []
    for i in range(batch):
        domain, seed = SIGNERS[i % 4]
        inputs.append(z.generate_app_inputs(_signed(2000 + i, domain, seed), spec, {"senderSalt": SALT + i, "recipient": i},
                                            params={"registry": reg}))
        assert inputs[-1]["registryIndex"] == str(SLOTS[i % 4])
        want.append(domain)
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    _, status = ctx.witness(b"".join(c.pack_inputs(x) for x in inputs), batch, want_witness=False)
    assert status == [-1] * batch
    proofs, publics, _ = ctx.prove(batch)
    npub = c.info.n_public
    js = [z.proof_to_json(proofs[256 * i:256 * (i + 1)], publics[32 * npub * i:32 * npub * (i + 1)], npub) for i in range(batch)]
    outs = [z.decode_app_outputs(spec, p) for _, p in js]
    assert {o["registryRoot"] for o in outs} == {reg.root}
    assert [o["dkimDomain"] for o in outs] == want
    assert z.Verifier(vk, device=0).verify_batch([p for _, p in js], [q for q, _ in js]) == [True] * batch

    # the key of corp78.com is not registered for alias77.org
    with pytest.raises(ValueError, match='domain "alias77.org"'):
        z.generate_app_inputs(_signed(5000, "alias77.org", 78), spec, {"senderSalt": SALT, "recipient": 0}, params={"registry": reg})
