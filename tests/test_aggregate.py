"""Groth16 proof aggregation on the host (no GPU): the oracle prover and verifier (oracle/aggregate.py), and the native
host verifier (zke_agg_verify / verify_aggregate) against the oracle's verdict.

  * the oracle aggregates and verifies at n = 2, 4, 8 on toy-key proofs and on re-randomised proof_of_twitter proofs;
  * it rejects a changed public signal, a proof swapped for a valid proof of other publics, a reordered batch, a cross
    term or folded value altered in any round, an altered opening and a verifier key from other taus - and the native
    verifier agrees on every case;
  * every refusal: n not a power of two, n above the SRS size, points off the curve or outside the subgroup, public
    signal counts that do not match the key.
"""
import pytest

import zkemail_b200 as z
from oracle import aggregate as ag
from oracle import bn254 as b

from agg_util import TAU_A, TAU_B, toy_batch, toy_proof, twitter_batch


def _native(vk, vkey, pubs, agg):
    return z.verify_aggregate(vk, vkey, pubs, agg)


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("source", ["toy", "twitter"])
def test_oracle_aggregates_and_verifies(n, source):
    if source == "toy":
        vkey, _, pubs, proofs = toy_batch(n)
    else:
        vkey, pubs, proofs = twitter_batch(n)
    srs = ag.Srs(TAU_A, TAU_B, n)
    agg = ag.aggregate(srs, vkey, proofs, pubs)
    assert len(agg) == ag.agg_bytes(n) == z._lib.zke_agg_bytes(n)
    assert ag.verify(srs.vk(), vkey, pubs, agg)
    assert _native(srs.vk(), vkey, pubs, agg) is True


@pytest.fixture(scope="module")
def batch4():
    vkey, sec, pubs, proofs = toy_batch(4)
    srs = ag.Srs(TAU_A, TAU_B, 4)
    return vkey, sec, pubs, proofs, srs, ag.aggregate(srs, vkey, proofs, pubs)


def _tampered(agg: bytes, off: int, new: bytes) -> bytes:
    return agg[:off] + new + agg[off + len(new):]


def _gt_at(agg, off):
    return ag.gt_from(agg[off:off + ag.GT_BYTES])


def _cases(batch4):
    vkey, sec, pubs, proofs, srs, agg = batch4
    vk = srs.vk()
    out = {}
    bad = [list(r) for r in pubs]
    bad[2][1] = (bad[2][1] + 1) % b.R
    out["changed public signal"] = (vk, bad, agg)
    other = [pubs[0], [5, 6], pubs[2], pubs[3]]
    import random
    swapped = list(proofs)
    swapped[1] = toy_proof(sec, other[1], random.Random(3))
    out["proof of other publics"] = (vk, pubs, ag.aggregate(srs, vkey, swapped, other))
    out["reordered batch"] = (vk, [pubs[1], pubs[0], pubs[2], pubs[3]], agg)
    for rnd in range(2):
        base = ag.HEAD_BYTES + rnd * ag.ROUND_BYTES
        sq = _gt_at(agg, base + 2 * ag.GT_BYTES)          # TL: replace by its square, still an element of GT
        out[f"round {rnd} TL"] = (vk, pubs, _tampered(agg, base + 2 * ag.GT_BYTES, ag.gt_b(sq * sq)))
        zcl = ag.g1_from(agg[base + 10 * ag.GT_BYTES:][:64])
        out[f"round {rnd} ZCL"] = (vk, pubs, _tampered(agg, base + 10 * ag.GT_BYTES, ag.g1_b(b.g1_add(zcl, b.G1_GEN))))
    fin = ag.HEAD_BYTES + 2 * ag.ROUND_BYTES
    fa = ag.g1_from(agg[fin:fin + 64])
    out["folded A"] = (vk, pubs, _tampered(agg, fin, ag.g1_b(b.g1_add(fa, b.G1_GEN))))
    fw1 = ag.g1_from(agg[fin + 512:fin + 576])
    out["folded w1"] = (vk, pubs, _tampered(agg, fin + 512, ag.g1_b(b.g1_add(fw1, b.G1_GEN))))
    op = len(agg) - 128
    pw1 = ag.g1_from(agg[op:op + 64])
    out["opening pi_w1"] = (vk, pubs, _tampered(agg, op, ag.g1_b(b.g1_add(pw1, b.G1_GEN))))
    pv2 = ag.g2_from(agg[op - 128:op])
    out["opening pi_v2"] = (vk, pubs, _tampered(agg, op - 128, ag.g2_b(b.g2_add(pv2, b.G2_GEN))))
    out["key of other taus"] = (ag.Srs(TAU_A + 1, TAU_B, 2).vk(), pubs, agg)
    z_ab = _gt_at(agg, 4 * ag.GT_BYTES)
    out["Z_AB"] = (vk, pubs, _tampered(agg, 4 * ag.GT_BYTES, ag.gt_b(z_ab * z_ab)))
    return vkey, out


def test_oracle_and_native_reject_every_tampering(batch4):
    vkey, cases = _cases(batch4)
    *_, srs, agg = batch4
    assert ag.verify(srs.vk(), vkey, batch4[2], agg) and _native(srs.vk(), vkey, batch4[2], agg)
    for name, (vk, pubs, bad) in cases.items():
        assert ag.verify(vk, vkey, pubs, bad) is False, name
        assert _native(vk, vkey, pubs, bad) is False, name


def test_refusals(batch4):
    vkey, sec, pubs, proofs, srs, agg = batch4
    vk = srs.vk()
    with pytest.raises(ag.AggError, match="power of two"):
        ag.aggregate(ag.Srs(TAU_A, TAU_B, 4), vkey, proofs[:3], pubs[:3])
    with pytest.raises(ag.AggError, match="exceed the SRS size"):
        ag.aggregate(ag.Srs(TAU_A, TAU_B, 2), vkey, proofs, pubs)
    with pytest.raises(ag.AggError, match="public signals"):
        ag.aggregate(srs, vkey, proofs, [p + [1] for p in pubs])
    for n in (3, 1, 16384):
        with pytest.raises(z._lib.ZkeError, match="power of two"):
            z.verify_aggregate(vk, vkey, (pubs * 4096)[:n], agg)
        assert not ag.verify(vk, vkey, (pubs * 4096)[:n], agg)
    with pytest.raises(z._lib.ZkeError, match="public signals"):
        z.verify_aggregate(vk, vkey, [p + [1] for p in pubs], agg)
    assert not ag.verify(vk, vkey, [p + [1] for p in pubs], agg)
    with pytest.raises(z._lib.ZkeError, match="bytes"):
        z.verify_aggregate(vk, vkey, pubs, agg[:-1])
    # a final A off the curve, a final B on the twist but outside the order-r subgroup
    fin = ag.HEAD_BYTES + 2 * ag.ROUND_BYTES
    off = _tampered(agg, fin, ag.fq_b(1) + ag.fq_b(1))
    with pytest.raises(z._lib.ZkeError, match="not on the curve"):
        z.verify_aggregate(vk, vkey, pubs, off)
    assert not ag.verify(vk, vkey, pubs, off)
    from test_pairing_emulation import _twist_point_outside_subgroup
    q = _twist_point_outside_subgroup()
    outside = _tampered(agg, fin + 64, ag.g2_b(q))
    with pytest.raises(z._lib.ZkeError, match="subgroup"):
        z.verify_aggregate(vk, vkey, pubs, outside)
    assert not ag.verify(vk, vkey, pubs, outside)
    unreduced = _tampered(agg, 0, b.P.to_bytes(32, "little"))
    with pytest.raises(z._lib.ZkeError, match="not reduced"):
        z.verify_aggregate(vk, vkey, pubs, unreduced)
    bad_vk = dict(vk, protocol="groth16")
    with pytest.raises(z._lib.ZkeError, match="snarkpack"):
        z.verify_aggregate(bad_vk, vkey, pubs, agg)

