"""Proof aggregation (SnarkPack, zk-email-verify_b200/csrc/aggregate.cu) against batch verification of the same proofs.

Proofs: GPU proofs of the Multiplier circuit (one public signal) under one toy key, made in batches of 512.  SRS: two
toy `.ptau` files of power 14 (independent known taus).  For n = 64, 512, 4096 and 8192: the wall time of `aggregate`
(GPU prover, one synchronous call incl. copies and the host quotients), of `verify_aggregate` (host verifier) and of
`Verifier.verify_batch_raw` (GPU batch verifier) over the same n proofs, each the median of `--repeats` calls after one
warm-up call, and the aggregate's size.  Every aggregate is asserted to verify.  Prints one JSON line, with the card's
name, power limit and SM clock read by nvidia-smi in the same run.

    python scripts/agg_bench.py [--repeats 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "zk-email-verify_b200", "host")):
    if p not in sys.path:
        sys.path.insert(0, p)

import zkemail_b200 as z  # noqa: E402


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _median_time(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("agg_bench needs a CUDA device")
    c = z.Circuit("Multiplier")
    zk = z.Zkey(c, seed=9, device=0)
    vkey = zk.vkey()
    batch, n_max = 512, 8192
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    proofs, publics = b"", b""
    for k in range(n_max // batch):
        packed = b"".join(c.pack_inputs({"a": 3 + i + batch * k, "b": 5 + 7 * i}) for i in range(batch))
        p, s, status = ctx.fullprove(packed, batch)
        assert status == [-1] * batch
        proofs, publics = proofs + p, publics + s
    ctx.close()
    npub = c.info.n_public
    t = time.perf_counter()
    srs = z.AggSrs.from_ptau(z.ptau_toy(14, 0x1234567, 3, 5), z.ptau_toy(14, 0x7654321, 7, 11), n_max=n_max)
    srs_s = time.perf_counter() - t
    agg_vk = srs.vk()
    ver = z.Verifier(vkey)
    rows = []
    for n in (64, 512, 4096, 8192):
        pb, sb = proofs[:256 * n], publics[:32 * npub * n]
        agg = z.aggregate(srs, vkey, pb, sb)
        assert z.verify_aggregate(agg_vk, vkey, sb, agg)
        t_agg = _median_time(lambda: z.aggregate(srs, vkey, pb, sb), args.repeats)
        t_ver = _median_time(lambda: z.verify_aggregate(agg_vk, vkey, sb, agg), args.repeats)
        t_batch = _median_time(lambda: ver.verify_batch_raw(pb, sb, n), args.repeats)
        rows.append({"n": n, "aggregate_s": round(t_agg, 4), "verify_aggregate_s": round(t_ver, 4),
                     "gpu_verify_batch_s": round(t_batch, 4), "aggregate_bytes": len(agg["aggregate"]) // 2,
                     "proof_bytes": 256 * n + 32 * npub * n})
        print(json.dumps(rows[-1]), file=sys.stderr)
    ver.close()
    srs.close()
    line = json.dumps({"bench": "agg_bench", "circuit": "Multiplier", "srs_from_ptau_s": round(srs_s, 3), "rows": rows,
                       **_gpu_info()})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
