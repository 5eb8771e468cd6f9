"""Groth16 proof aggregation on the GPU (`-m gpu`): zk-email-verify_b200/csrc/aggregate.cu through AggSrs / aggregate.

  * the SRS read from two toy `.ptau` files equals the oracle's SRS of the same secrets (verifier key);
  * at n = 8 the device aggregate equals the oracle's byte for byte (the transcript is deterministic);
  * 64 GPU proofs of EmailVerifier(640, 768) aggregate on the device and verify under the native and the oracle
    verifiers; tampering with one of those proofs makes verification fail;
  * the device prover's refusals: n, SRS size, a proof point outside its group, the .ptau pair.
"""
import pytest

import zkemail_b200 as z
from oracle import aggregate as ag
from oracle import bn254 as b

from agg_util import TAU_A, TAU_B, proofs256, publics_bytes, toy_batch
from test_pairing_emulation import _twist_point_outside_subgroup

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ptaus():
    return z.ptau_toy(5, TAU_A, 3, 5), z.ptau_toy(5, TAU_B, 7, 11)


def test_device_aggregate_equals_oracle_at_8(ptaus):
    srs = z.AggSrs.from_ptau(*ptaus, n_max=8)
    ref = ag.Srs(TAU_A, TAU_B, 8)
    assert srs.vk() == ref.vk()
    vkey, _, pubs, proofs = toy_batch(8)
    got = z.aggregate(srs, vkey, [{"pi_a": b.g1_to_json(p[0]), "pi_b": b.g2_to_json(p[1]), "pi_c": b.g1_to_json(p[2])}
                                  for p in proofs], pubs)
    want = ag.aggregate(ref, vkey, proofs, pubs)
    assert bytes.fromhex(got["aggregate"]) == want
    assert got["n"] == 8 and z.verify_aggregate(srs.vk(), vkey, pubs, got)
    # the raw layout gives the same bytes
    assert z.aggregate(srs, vkey, proofs256(proofs), publics_bytes(pubs))["aggregate"] == got["aggregate"]
    srs.close()


def test_device_refusals(ptaus):
    srs = z.AggSrs.from_ptau(*ptaus, n_max=4)
    vkey, _, pubs, proofs = toy_batch(8)
    with pytest.raises(z._lib.ZkeError, match="exceed the SRS size"):
        z.aggregate(srs, vkey, proofs256(proofs), publics_bytes(pubs))
    with pytest.raises(z._lib.ZkeError, match="power of two"):
        z.aggregate(srs, vkey, proofs256(proofs[:3]), publics_bytes(pubs[:3]))
    bad = bytearray(proofs256(proofs[:4]))
    bad[256 + 64:256 + 192] = ag.g2_b(_twist_point_outside_subgroup())
    with pytest.raises(z._lib.ZkeError, match="proof 1"):
        z.aggregate(srs, vkey, bytes(bad), publics_bytes(pubs[:4]))
    bad = bytearray(proofs256(proofs[:4]))
    bad[2 * 256:2 * 256 + 64] = ag.fq_b(1) + ag.fq_b(1)
    with pytest.raises(z._lib.ZkeError, match="proof 2"):
        z.aggregate(srs, vkey, bytes(bad), publics_bytes(pubs[:4]))
    srs.close()
    with pytest.raises(z._lib.ZkeError, match="too small"):
        z.AggSrs.from_ptau(*ptaus, n_max=32)
    with pytest.raises(z._lib.ZkeError, match="independent"):
        z.AggSrs.from_ptau(ptaus[0], ptaus[0], n_max=4)


def test_email_verifier_64_gpu_proofs(ptaus):
    c = z.Circuit("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1])
    key = z.synthetic.generate_key()
    inputs = []
    for i in range(4):
        email = z.synthetic.make_signed_email(i, key, body_len=512)
        dk = z.verify_dkim_signature(email, resolver=lambda n, t: [z.synthetic.key_record(key)])
        inputs.append(z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": 640, "maxBodyLength": 768}))
    zk = z.Zkey(c, seed=3, device=0)
    vkey = zk.vkey()
    n = 64
    ctx = z.Context(c, zk, device=0, max_batch=n)
    packed = b"".join(c.pack_inputs(inputs[k % 4]) for k in range(n))
    proofs, publics, status = ctx.fullprove(packed, n)
    assert status == [-1] * n
    ctx.close()
    srs = z.AggSrs.from_ptau(z.ptau_toy(7, TAU_A, 3, 5), z.ptau_toy(7, TAU_B, 7, 11), n_max=64)
    agg = z.aggregate(srs, vkey, proofs, publics)
    assert z.verify_aggregate(srs.vk(), vkey, publics, agg)
    npub = c.info.n_public
    pubs = [[int.from_bytes(publics[32 * (npub * k + j):32 * (npub * k + j + 1)], "little") for j in range(npub)] for k in range(n)]
    assert ag.verify(srs.vk(), vkey, pubs, bytes.fromhex(agg["aggregate"]))
    # one proof tampered: its C moved by the generator - the aggregate of the batch no longer verifies
    bad = bytearray(proofs)
    k = 37
    c_k = ag.g1_from(bytes(bad[256 * k + 192:256 * k + 256]))
    bad[256 * k + 192:256 * k + 256] = ag.g1_b(b.g1_add(c_k, b.G1_GEN))
    bad_agg = z.aggregate(srs, vkey, bytes(bad), publics)
    assert not z.verify_aggregate(srs.vk(), vkey, publics, bad_agg)
    assert not ag.verify(srs.vk(), vkey, pubs, bytes.fromhex(bad_agg["aggregate"]))
    srs.close()
