"""Circuits read from circom's `.r1cs` on the GPU: key setup from a `.ptau` and contributions against the CPU oracle, the key
audit, `wtns check`, proving from `.wtns`, and at EmailVerifier scale the same keys, checks and proofs as the template
circuit the file was written from."""
import ctypes

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkemail_b200.iden3_binfile import write_wtns
from zkutil import oracle_prove, oracle_setup, product_sections, ref, ref_view
from oracle import bn254
from test_r1cs_reader import R, synthetic, synthetic_file, tampered, witness_bytes

pytestmark = pytest.mark.gpu

TOX = (0x1F2E3D4C5B6A79880123456789ABCDEF0FEDCBA98765432, 0x2468ACE013579BDF2468ACE013579BDF, 0x0DDBA11CAFEBABE5EED)
S1 = 0x5EC2E7 * 10 ** 30 + 17
RS = (0x1234567890ABCDEF1234567890ABCDEF, 0xFEDCBA0987654321FEDCBA0987654321)


def _le(x):
    return int(x).to_bytes(32, "little")


@pytest.fixture(scope="module")
def syn():
    s = synthetic()
    return s, z.Circuit.from_r1cs(synthetic_file(s))


@pytest.fixture(scope="module")
def ptau10():
    return z.ptau_toy(10, *TOX)


@pytest.fixture(scope="module")
def key(syn, ptau10):
    return z.Zkey.from_ptau(syn[1], ptau10).contribute(_le(S1))


def _other_key(ptau10):
    """A key for the same-shaped synthetic R1CS with one A coefficient changed."""
    other = z.Circuit.from_r1cs(synthetic_file(synthetic(tweak=True)))
    return other, z.Zkey.from_ptau(other, ptau10).contribute(_le(S1))


def test_setup_and_contribution_equal_the_oracle(syn, ptau10):
    _, c = syn
    assert c.info.domain_log2 + 1 <= 10
    base = z.Zkey.from_ptau(c, ptau10)
    assert product_sections(base) == oracle_setup(c, TOX + (1, 1)), "from_ptau differs from the oracle setup at gamma = delta = 1"
    k1 = base.contribute(_le(S1))
    assert product_sections(k1) == oracle_setup(c, TOX + (1, S1))
    assert k1.check_contribution(base)


def test_verify_zkey(syn, ptau10, key):
    _, c = syn
    assert z.verify_zkey(c, ptau10, key)
    _, other = _other_key(ptau10)
    assert not z.verify_zkey(c, ptau10, other)


def test_check_wtns_and_prove_equal_the_oracle(syn, key):
    s, c = syn
    ctx = z.Context(c, key, device=0, max_batch=1)
    good = witness_bytes(s["witness"])
    assert ctx.check_wtns(write_wtns(good)) == -1
    bad = witness_bytes(tampered(s, 40))
    want = ref.zkref_check_r1cs(ctypes.byref(ref_view(c)), bad)
    assert want == 40
    assert ctx.check_wtns(write_wtns(bad), raise_on_fail=False) == want
    with pytest.raises(z.AssertFailed, match="Assert Failed: constraint 40 "):
        ctx.check_wtns(write_wtns(bad))
    proof, publics = ctx.wtns_prove(write_wtns(good), _le(RS[0]) + _le(RS[1]))
    ctx.close()
    assert proof == oracle_prove(c, product_sections(key), good, RS[0], RS[1])
    n_pub = c.info.n_public
    assert publics == b"".join(_le(v) for v in s["witness"][1:1 + n_pub])
    pj, pubs = z.proof_to_json(proof, publics, n_pub)
    vk = key.vkey()
    assert bn254.groth16_verify(vk, pubs, pj) and z.verify(vk, pubs, pj)
    assert z.Verifier(vk).verify_batch([pubs], [pj]) == [True]


def test_loaded_key_is_checked_against_the_circuit(syn, ptau10, key):
    s, c = syn
    loaded = z.Zkey.load(key.write(), circuit=c)
    ctx = z.Context(c, loaded, device=0, max_batch=1)       # the same system: accepted
    assert ctx.check_wtns(write_wtns(witness_bytes(s["witness"]))) == -1
    ctx.close()
    _, other = _other_key(ptau10)
    foreign = z.Zkey.load(other.write())
    with pytest.raises(L.ZkeError, match="zkey does not belong to this circuit: A row 0 differs"):
        z.Context(c, foreign, device=0, max_batch=1)
    key_only = z.Context(None, foreign, device=0, max_batch=1)
    key_only.load_witness(witness_bytes(s["witness"]), 1)
    with pytest.raises(L.ZkeError, match="no C matrix"):
        key_only.check_witness(1)
    key_only.close()


def test_context_without_a_key(syn, key):
    s, c = syn
    ctx = z.Context(c, device=0, max_batch=2)
    good, bad = witness_bytes(s["witness"]), witness_bytes(tampered(s, 7))
    ctx.load_witness(good + bad, 2)
    assert ctx.check_witness(2, raise_on_fail=False) == [-1, 7]
    ctx.load_witness(good + good, 2)
    assert ctx.check_witness(2) == [-1, -1]
    inputs = bytes(32 * c.n_inputs)
    msg = "this circuit was read from an .r1cs: it has no witness program"
    with pytest.raises(L.ZkeError, match=msg):
        ctx.witness(inputs, 1)
    with pytest.raises(L.ZkeError, match=msg):
        ctx.upload_inputs(inputs, 1)
    ctx.close()
    ctx = z.Context(c, key, device=0, max_batch=1)
    with pytest.raises(L.ZkeError, match=msg):
        ctx.fullprove(inputs, 1)
    with pytest.raises(L.ZkeError, match=msg):
        ctx.submit(inputs, 1)
    ctx.close()


# ------------------------------------------------------------------------------------------------ EmailVerifier scale
def _resolver(k):
    return lambda n, t: [z.synthetic.key_record(k)]


def test_email_verifier_from_r1cs_matches_the_template_circuit():
    """EmailVerifier(640, 768), N = 2^21, with the seeded toy setup (no 4 GB .ptau needed): the circuit read back from its
    own `.r1cs` gives the same key, accepts and rejects the same witnesses and proves the same proofs."""
    c = z.Circuit("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1])
    rc = z.Circuit.from_r1cs(c.write_r1cs())
    seed = 91
    toy, toy_r = z.Zkey(c, seed=seed), z.Zkey(rc, seed=seed)
    assert product_sections(toy_r) == product_sections(toy)
    del toy_r
    k = z.synthetic.generate_key(seed=5)
    inputs = []
    for i in range(4):
        dk = z.verify_dkim_signature(z.synthetic.make_signed_email(30 + i, k, body_len=512), resolver=_resolver(k))
        inputs.append(z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": 640, "maxBodyLength": 768}))
    ctx_t = z.Context(c, toy, device=0, max_batch=4)
    wt, status = ctx_t.witness(b"".join(c.pack_inputs(x) for x in inputs), 4)
    assert status == [-1] * 4
    ctx_r = z.Context(rc, toy, device=0, max_batch=4)
    ctx_r.load_witness(wt, 4)
    assert ctx_r.check_witness(4) == [-1] * 4
    m = c.info.n_vars
    bad = bytearray(wt)
    wire = m - 5
    off = 32 * (2 * m + wire)
    bad[off:off + 32] = _le((int.from_bytes(wt[off:off + 32], "little") + 1) % R)
    ctx_t.load_witness(bytes(bad), 4)
    want = ctx_t.check_witness(4, raise_on_fail=False)
    assert want[2] >= 0 and want[:2] + want[3:] == [-1] * 3
    ctx_r.load_witness(bytes(bad), 4)
    assert ctx_r.check_witness(4, raise_on_fail=False) == want
    rs = b"".join(_le(RS[0] + e) + _le(RS[1] + e) for e in range(4))
    ctx_t.load_witness(wt, 4)
    ctx_r.load_witness(wt, 4)
    assert ctx_r.prove(4, rs)[:2] == ctx_t.prove(4, rs)[:2]
    ctx_t.close()
    ctx_r.close()
