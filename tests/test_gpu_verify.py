"""GPU batch verifier (`-m gpu`): zk-email-verify_b200/csrc/verify.cu through zke_verifier_* / Verifier.

  * the device pairing (zke_selftest_pairing_gpu) equals the host's zke_pairing_alphabeta on random pairs and on the
    proof_of_twitter fixture's alpha / beta;
  * every case of the host batch verifier's tests (tests/test_verifier_fixture.py), rebuilt as one mixed batch, gets the
    host's per-proof verdicts with the same weights, and n = 0 / n = 1;
  * proofs made by Context.prove verify through verify_batch_raw, also tiled past block and grid boundaries, and a
    corrupted entry is named;
  * zke_verifier_open refuses bad keys; argument errors raise ValueError.
"""
import ctypes
import json
import os
import random

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from oracle import bn254

from test_verifier_fixture import Q, R_ORDER, _load, _rerandomised
from test_pairing_emulation import _twist_point_outside_subgroup

pytestmark = pytest.mark.gpu

le = lambda v: int(v).to_bytes(32, "little")


def _g1b(p):
    return le(p[0]) + le(p[1])


def _g2b(q):
    return le(q[0][0]) + le(q[0][1]) + le(q[1][0]) + le(q[1][1])


def _gpu_pairings(pairs):
    n = len(pairs)
    out = ctypes.create_string_buffer(384 * n)
    err = ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_selftest_pairing_gpu(0, n, b"".join(_g1b(p) for p, _ in pairs), b"".join(_g2b(q) for _, q in pairs), out, err, L.ERRCAP)
    assert rc == 0, err.value
    return [out.raw[384 * i:384 * (i + 1)] for i in range(n)]


def _host_pairing(p, q):
    out = ctypes.create_string_buffer(384)
    assert L.zke_pairing_alphabeta(_g1b(p), _g2b(q), out) == 0
    return out.raw


def test_gpu_pairing_matches_host_pairing():
    rng = random.Random(21)
    pairs = [(bn254.g1_mul(bn254.G1_GEN, rng.randrange(1, R_ORDER)), bn254.g2_mul(bn254.G2_GEN, rng.randrange(1, R_ORDER)))
             for _ in range(10)]
    vkey, _, _ = _load()
    pairs.append((bn254.g1_from_json(vkey["vk_alpha_1"]), bn254.g2_from_json(vkey["vk_beta_2"])))
    got = _gpu_pairings(pairs)
    for (p, q), g in zip(pairs, got):
        assert g == _host_pairing(p, q)
    ab = [[[str(int.from_bytes(got[-1][32 * ((i * 3 + j) * 2 + k):32 * ((i * 3 + j) * 2 + k) + 32], "little")) for k in range(2)]
           for j in range(3)] for i in range(2)]
    assert ab == vkey["vk_alphabeta_12"]


def _mixed_batch():
    """The cases of test_verifier_fixture's batch tests as one list of (public signals, proof)."""
    vkey, public, proof = _load()
    good = [proof, _rerandomised(proof, 7), _rerandomised(proof, 0x1234567890abcdef)]
    items = [(public, p) for p in good]
    bad_c = json.loads(json.dumps(proof))
    bad_c["pi_c"][1] = str(Q - int(bad_c["pi_c"][1]))
    items.append((public, bad_c))
    bad_pub = list(public)
    bad_pub[1] = str(int(bad_pub[1]) + 1)
    items.append((bad_pub, good[1]))
    d = bn254.g1_mul((1, 2), 5)
    p0, p1 = json.loads(json.dumps(proof)), json.loads(json.dumps(good[1]))
    p0["pi_c"] = bn254.g1_to_json(bn254.g1_add(bn254.g1_from_json(proof["pi_c"]), d))
    p1["pi_c"] = bn254.g1_to_json(bn254.g1_add(bn254.g1_from_json(good[1]["pi_c"]), bn254.g1_neg(d)))
    items += [(public, p0), (public, p1)]
    off = json.loads(json.dumps(proof))
    off["pi_a"][0] = str(int(off["pi_a"][0]) + 1)
    items.append((public, off))
    rogue_b = _twist_point_outside_subgroup()
    rogue = json.loads(json.dumps(proof))
    rogue["pi_b"] = [[str(rogue_b[0][0]), str(rogue_b[0][1])], [str(rogue_b[1][0]), str(rogue_b[1][1])], ["1", "0"]]
    items.append((public, rogue))
    items.append((public[:-1], proof))                       # wrong number of public signals
    items.append((public + ["1"], proof))
    big = list(public)
    big[0] = str(int(big[0]) + R_ORDER)                      # a public signal >= r
    items.append((big, proof))
    inf_a = json.loads(json.dumps(proof))
    inf_a["pi_a"] = ["0", "1", "0"]                          # infinity points (z = 0): valid encodings, wrong proof
    items.append((public, inf_a))
    inf_b = json.loads(json.dumps(proof))
    inf_b["pi_b"] = [["0", "0"], ["1", "0"], ["0", "0"]]
    items.append((public, inf_b))
    inf_c = json.loads(json.dumps(proof))
    inf_c["pi_c"] = ["0", "1", "0"]
    items.append((public, inf_c))
    return vkey, items


def test_mixed_batch_matches_host_verdicts():
    vkey, items = _mixed_batch()
    v = z.Verifier(vkey)
    sigs, proofs = [s for s, _ in items], [p for _, p in items]
    rng = random.Random(5)
    rand = bytes(rng.getrandbits(8) for _ in range(16 * len(items)))
    host = z.verify_batch(vkey, sigs, proofs, rand=rand)
    assert host[:3] == [True] * 3 and not any(host[3:])
    assert v.verify_batch(sigs, proofs, rand=rand) == host
    assert v.verify_batch(sigs, proofs) == host                           # library-drawn weights
    # the valid members alone pass the combined check; each case alone gives the host's verdict (n = 1)
    assert v.verify_batch(sigs[:3], proofs[:3], rand=rand[:48]) == [True] * 3
    for k in range(len(items)):
        assert v.verify_batch([sigs[k]], [proofs[k]]) == z.verify_batch(vkey, [sigs[k]], [proofs[k]]), f"case {k}"
    # errors that cancel under equal weights (cases 5 and 6) are caught by distinct weights; with equal weights both
    # verifiers are fooled alike
    assert v.verify_batch(sigs[5:7], proofs[5:7], rand=rand[:32]) == [False, False]
    equal = bytes([1] + [0] * 15) * 2
    assert v.verify_batch(sigs[5:7], proofs[5:7], rand=equal) == z.verify_batch(vkey, sigs[5:7], proofs[5:7], rand=equal) == [True, True]
    assert v.verify_batch([], []) == []
    v.close()


def test_gpu_made_proofs_verify_raw_and_tiled():
    c = z.Circuit("Multiplier")
    zk = z.Zkey(c, seed=9, device=0)
    batch = 8
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    packed = b"".join(c.pack_inputs({"a": 3 + k, "b": 5 + 7 * k}) for k in range(batch))
    proofs, publics, status = ctx.fullprove(packed, batch)
    assert status == [-1] * batch
    v = z.Verifier(zk.vkey())
    assert v.verify_batch_raw(proofs, publics, batch) == [True] * batch
    reps = 4096 // batch + 3                                  # 4120 entries: not a multiple of the block or fold sizes
    n = batch * reps
    big_p, big_s = proofs * reps, publics * reps
    assert v.verify_batch_raw(big_p, big_s, n) == [True] * n
    bad = bytearray(big_s)
    k = 2345
    bad[32 * c.info.n_public * k] ^= 1                       # one public signal of entry k
    got = v.verify_batch_raw(big_p, bytes(bad), n)
    assert got[k] is False and sum(got) == n - 1
    ctx.close()
    v.close()


def test_open_refuses_bad_keys():
    vkey, _, _ = _load()
    off = json.loads(json.dumps(vkey))
    off["vk_alpha_1"][0] = str(int(off["vk_alpha_1"][0]) + 1)
    off_ic = json.loads(json.dumps(vkey))
    off_ic["IC"][1][1] = str(int(off_ic["IC"][1][1]) + 1)
    rogue_b = _twist_point_outside_subgroup()
    rogue = [[str(rogue_b[0][0]), str(rogue_b[0][1])], [str(rogue_b[1][0]), str(rogue_b[1][1])], ["1", "0"]]
    bad_gamma, bad_delta = json.loads(json.dumps(vkey)), json.loads(json.dumps(vkey))
    bad_gamma["vk_gamma_2"], bad_delta["vk_delta_2"] = rogue, rogue
    for bad, msg in ((off, "vk_alpha_1"), (off_ic, "IC"), (bad_gamma, "vk_gamma_2"), (bad_delta, "vk_delta_2")):
        with pytest.raises(L.ZkeError, match=msg):
            z.Verifier(bad)


def test_argument_errors():
    vkey, public, proof = _load()
    v = z.Verifier(vkey)
    with pytest.raises(ValueError):
        v.verify_batch([public], [proof, proof])
    with pytest.raises(ValueError):
        v.verify_batch([public], [proof], rand=b"short")
    with pytest.raises(ValueError):
        v.verify_batch_raw(bytes(256), bytes(32 * v.n_public), 2)
    with pytest.raises(ValueError):
        v.verify_batch_raw(bytes(256), bytes(32 * v.n_public), 1, rand=bytes(8))
    v.close()
