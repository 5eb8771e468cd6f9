"""The key registry on the GPU: zke_poseidon_batch against the host permutation, zke_pubkey_hashes against
poseidon_large, zke_merkle_build against oracle/merkle.py level for level, then an app with `"keyRegistryDepth"`: its
GPU witness against the CPU oracle bit for bit (cluster widths default, 1 and 8, native Poseidon on and off), its proof
at fixed (r, s) against the oracle's under every verifier, and a batch of 64 emails signed by four keys of a 1,000-key
registry proved under one key, every proof publishing the same root."""
import ctypes
import functools
import random

import pytest

import zkemail_b200 as z
import zkutil
from oracle import merkle
from test_app_commit import SALT, commit_body, commit_spec
from zkutil import oracle_witness

pytestmark = pytest.mark.gpu

R = z.FR_MODULUS
L = z._lib
DEPTH = 10
N_KEYS = 1000
KEY_SEEDS = [77, 78, 79, 80]
KEY_SLOTS = [0, 333, 998, 999]       # where the four signing keys sit among the 1,000


def _host_hash(row):
    out = ctypes.create_string_buffer(32)
    assert L.zke_poseidon_hash(b"".join(x.to_bytes(32, "little") for x in row), len(row), out) == 0
    return int.from_bytes(out.raw, "little")


@pytest.mark.parametrize("width", range(1, 17))
def test_poseidon_batch_matches_host(width):
    """Every instance at counts up to 1,000; at 65,537 every instance for widths 1..3 and every 61st (plus the ends)
    above, where the host permutation would take minutes."""
    rng = random.Random(width)
    for count in (1, 31, 32, 33, 1000, 65537):
        rows = [[rng.randrange(R) for _ in range(width)] for _ in range(count)]
        rows[0] = [0] * width
        rows[-1] = [R - 1] * width
        got = z.hash.poseidon_batch(rows)
        check = range(count) if count <= 1000 or width <= 3 else sorted(set(range(0, count, 61)) | {count - 2, count - 1})
        for i in check:
            assert got[i] == _host_hash(rows[i]), (width, count, i)


def test_poseidon_batch_refuses_input_not_below_r():
    rows = [[1, 2]] * 40
    data = bytearray(b"".join(x.to_bytes(32, "little") for r in rows for x in r))
    data[32 * (2 * 37 + 1):32 * (2 * 37 + 2)] = R.to_bytes(32, "little")
    out, err = ctypes.create_string_buffer(32 * 40), ctypes.create_string_buffer(L.ERRCAP)
    assert L.zke_poseidon_batch(bytes(data), 2, 40, 0, out, err, L.ERRCAP) < 0
    assert b"instance 37" in err.value


def test_pubkey_hashes_match_poseidon_large():
    rng = random.Random(5)
    moduli = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(1000)]
    moduli[1] = (1 << 2057) - 1                                      # the largest value below 2^(n k)
    got = z.registry.pubkey_hashes(moduli)
    assert got == [z.hash.poseidon_large(m, 9, 242) for m in moduli]
    with pytest.raises(L.ZkeError, match="modulus 2 is not below 2"):
        z.registry.pubkey_hashes(moduli[:2] + [1 << 2057])
    key = z.synthetic.generate_key(seed=77)
    rec = z.synthetic.key_record(key)
    assert z.registry.pubkey_hashes([rec]) == [z.hash.poseidon_large(key.public_key().public_numbers().n, 9, 242)]


@pytest.mark.parametrize("m", [1, 2, 3, 255, 256, 257, 4097])
def test_merkle_build_matches_oracle(m):
    rng = random.Random(m)
    leaves = [rng.randrange(R) for _ in range(m)]
    leaves[0] = R - 1
    if m > 1:
        leaves[-1] = 0
    want = merkle.levels(leaves, 32)              # levels 0..d of a depth-d tree are the first d + 1 of this one
    for depth in (13, 20, 32):
        assert z.registry.merkle_levels(leaves, depth) == want[:depth + 1]
    if m <= 2:
        assert z.registry.merkle_levels(leaves, 1) == merkle.levels(leaves, 1)
    if m == 257:
        bad = leaves[:]
        bad[200] = R
        with pytest.raises(L.ZkeError, match="leaf 200 is not below r"):
            z.registry.merkle_levels(bad, 13)


# ---- the app -----------------------------------------------------------------------------------------------------------

_APP = {}


_key = functools.lru_cache(maxsize=None)(lambda seed: z.synthetic.generate_key(seed=seed))


def _signed(i, seed):
    key = _key(seed)
    em = z.synthetic.make_signed_email(i, key, domain=f"corp{seed}.com", body_override=commit_body(str(1000 + i), "a note"))
    return z.verify_dkim_signature(em, resolver=lambda n, t: [z.synthetic.key_record(key)]), key


def _app():
    if not _APP:
        spec = dict(commit_spec(1), keyRegistryDepth=DEPTH)
        c = z.Circuit.from_spec(spec)
        rng = random.Random(9)
        keys = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(N_KEYS)]
        dks = []
        for slot, seed in zip(KEY_SLOTS, KEY_SEEDS):
            dk, key = _signed(slot, seed)
            keys[slot] = z.synthetic.key_record(key)           # DKIM records and plain moduli side by side
            dks.append(dk)
        reg = z.KeyRegistry.build(keys, DEPTH)
        assert reg.root == merkle.root(reg.leaves, DEPTH)
        assert z.KeyRegistry.from_json(reg.to_json()).levels == reg.levels
        inputs = [z.generate_app_inputs(dk, spec, {"senderSalt": SALT + k, "recipient": k}, params={"registry": reg})
                  for k, dk in enumerate(dks)]
        _APP.update(spec=spec, c=c, reg=reg, dks=dks, inputs=inputs, refs=[oracle_witness(c, x).raw() for x in inputs])
    return _APP


@pytest.mark.parametrize("native", ["1", "0"], ids=["native", "gadget"])
@pytest.mark.parametrize("width", ["default", "1", "8"])
def test_registry_witness_matches_oracle(width, native, monkeypatch):
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


def test_registry_proofs(monkeypatch):
    from oracle import bn254
    monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    monkeypatch.delenv("ZKE_NATIVE_POSEIDON", raising=False)
    a = _app()
    c, spec, reg = a["c"], a["spec"], a["reg"]
    zk = z.Zkey(c, seed=23)
    vk = zk.vkey()

    ctx = z.Context(c, zk, device=0, max_batch=1)
    wt, status = ctx.witness(c.pack_inputs(a["inputs"][1]), 1)
    assert status == [-1] and wt == a["refs"][1]
    r, s = 515151, 626262
    proofs, publics, _ = ctx.prove(1, r.to_bytes(32, "little") + s.to_bytes(32, "little"))
    assert proofs == zkutil.oracle_prove(c, zkutil.product_sections(zk), wt, r, s)
    proof, pubs = z.proof_to_json(proofs, publics, c.info.n_public)
    assert bn254.groth16_verify(vk, pubs, proof) and z.verify(vk, pubs, proof)
    assert z.Verifier(vk, device=0).verify_batch([pubs], [proof]) == [True]
    assert z.verify_batch(vk, [pubs], [proof]) == [True]
    assert z.decode_app_outputs(spec, pubs)["registryRoot"] == reg.root
    del ctx

    # 64 emails, 16 per signing key, one proving key: every proof publishes the same root and verifies
    batch = 64
    inputs = []
    for i in range(batch):
        slot, seed = KEY_SLOTS[i % 4], KEY_SEEDS[i % 4]
        dk, _ = _signed(2000 + i, seed)
        inputs.append(z.generate_app_inputs(dk, spec, {"senderSalt": SALT + i, "recipient": i}, params={"registry": reg}))
        assert inputs[-1]["registryIndex"] == str(slot)
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    _, status = ctx.witness(b"".join(c.pack_inputs(x) for x in inputs), batch, want_witness=False)
    assert status == [-1] * batch
    proofs, publics, _ = ctx.prove(batch)
    npub = c.info.n_public
    js = [z.proof_to_json(proofs[256 * i:256 * (i + 1)], publics[32 * npub * i:32 * npub * (i + 1)], npub) for i in range(batch)]
    roots = {z.decode_app_outputs(spec, p)["registryRoot"] for _, p in js}
    assert roots == {reg.root}
    assert z.Verifier(vk, device=0).verify_batch([p for _, p in js], [q for q, _ in js]) == [True] * batch
