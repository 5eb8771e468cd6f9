"""Throughput of the GPU batch verifier (zkemail_b200.Verifier, zk-email-verify_b200/csrc/verify.cu).

64 distinct valid proofs of the proof_of_twitter fixture (tests/golden/proof_of_twitter), made by re-randomising
(k A, k^-1 B, C), are tiled to n = 64, 1024 and 16384 entries and checked with Verifier.verify_batch_raw: the median
wall time of `--repeats` synchronous calls after one warm-up call each, proofs/s = n / median.  The call includes the
host-to-device copies and the weight draw.  Also timed: n = 1024 with one bad proof (the combined check fails and every
proof is verified on its own) and the host verifier (verify_batch, zke_verify_batch_json) at n = 64.  Prints one JSON
line, with the card's name, power limit and SM clock read by nvidia-smi in the same run.

    python scripts/verify_bench.py [--repeats 5] [--out FILE]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "zk-email-verify_b200", "host")):
    if p not in sys.path:
        sys.path.insert(0, p)

import zkemail_b200 as z  # noqa: E402
from oracle import bn254  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "proof_of_twitter")


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _proofs(count, seed=1):
    vkey, public, proof = (json.load(open(os.path.join(GOLD, n))) for n in ("vkey.json", "public.json", "proof.json"))
    rng = random.Random(seed)
    a, b, c = bn254.g1_from_json(proof["pi_a"]), bn254.g2_from_json(proof["pi_b"]), bn254.g1_from_json(proof["pi_c"])
    le = lambda v: int(v).to_bytes(32, "little")
    raw, jsons = [], []
    for i in range(count):
        k = 1 if i == 0 else rng.randrange(2, bn254.R)
        ka, kb = bn254.g1_mul(a, k), bn254.g2_mul(b, pow(k, -1, bn254.R))
        raw.append(le(ka[0]) + le(ka[1]) + le(kb[0][0]) + le(kb[0][1]) + le(kb[1][0]) + le(kb[1][1]) + le(c[0]) + le(c[1]))
        pj = json.loads(json.dumps(proof))
        pj["pi_a"], pj["pi_b"] = bn254.g1_to_json(ka), bn254.g2_to_json(kb)
        jsons.append(pj)
    pub = b"".join(le(s) for s in public)
    return vkey, public, raw, jsons, pub


def _median_time(fn, repeats):
    fn()                                    # warm-up
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("verify_bench needs a CUDA device")
    vkey, public, raw, jsons, pub = _proofs(64)
    v = z.Verifier(vkey)
    res = {"metric": "groth16_verify_proofs_per_s", "circuit": "proof_of_twitter", "n_public": v.n_public}
    for n in (64, 1024, 16384):
        proofs = b"".join(raw[i % 64] for i in range(n))
        pubs = pub * n
        got = v.verify_batch_raw(proofs, pubs, n)
        assert all(got), "a valid proof was rejected"
        t = _median_time(lambda: v.verify_batch_raw(proofs, pubs, n), args.repeats)
        res[f"gpu_n{n}_ms"] = round(t * 1e3, 3)
        res[f"gpu_n{n}_proofs_per_s"] = round(n / t, 1)
    # n = 1024 with one bad proof: the per-proof path
    n = 1024
    bad = bytearray(b"".join(raw[i % 64] for i in range(n)))
    bad[256 * 517 + 192] ^= 1                # C.x of entry 517: off the curve
    bad = bytes(bad)
    got = v.verify_batch_raw(bad, pub * n, n)
    assert got[517] is False and sum(got) == n - 1
    t = _median_time(lambda: v.verify_batch_raw(bad, pub * n, n), args.repeats)
    res["gpu_n1024_one_bad_ms"] = round(t * 1e3, 3)
    res["gpu_n1024_one_bad_proofs_per_s"] = round(n / t, 1)
    # the host verifier at n = 64
    sigs = [public] * 64
    assert z.verify_batch(vkey, sigs, jsons) == [True] * 64
    t = _median_time(lambda: z.verify_batch(vkey, sigs, jsons), max(1, args.repeats // 2))
    res["host_n64_ms"] = round(t * 1e3, 3)
    res["host_n64_proofs_per_s"] = round(64 / t, 1)
    res.update(_gpu_info())
    v.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
