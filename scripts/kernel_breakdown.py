#!/usr/bin/env python
"""Per-kernel GPU time of the headline workload, from torch.profiler (CUPTI also records the kernels that the
ctypes-loaded engine library launches).

The context is built as bench.py builds it: default circuit, KEY_SEED proving key, a batch of 64 emails signed with the
seeded RSA key, seeded blinding scalars, inputs resident on the device.  The pipelined zke_fullprove_submit / _collect
loop runs under the profiler twice:
  lanes=8 : the steady state bench.py times (proofs of the batch overlap on eight lanes)
  lanes=1 : one lane, so that each kernel's time is close to its standalone time
For every kernel name: GPU time per proof, launches per proof, and that time as a share of the step's wall time per
proof.  Under overlap the shares add up to more than 1.  The card's name, power limit and SM clocks are read with
nvidia-smi in the same run.

  python scripts/kernel_breakdown.py [--steps 2] [--warmup 2] [--top 40] [--json OUT]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (sets up the package path; workload constants and input helpers)


def short_name(name):
    """'void zke::dev::chunk_sum_kernel<zke::dev::Fq, 5>(unsigned char const*, ...)' -> 'chunk_sum_kernel<Fq, 5>'"""
    name = re.sub(r"^void ", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):       # drop the argument list (the first '(' outside template brackets)
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return re.sub(r"\b(zke::dev::|zke::|\(anonymous namespace\)::)", "", name[:cut])


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=10)
    return dict(zip(q.split(","), [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")])) if out.stdout.strip() else {}


def profile_run(torch, ctx, batch, rs, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        ctx.submit(None, batch, rs)
        for _ in range(steps - 1):
            ctx.submit(None, batch, rs)
            ctx.collect()
        _, _, status = ctx.collect()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    assert status == [-1] * batch, status
    per = defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0 and not ev.name.startswith("Memcpy") \
                and not ev.name.startswith("Memset"):
            k = per[short_name(ev.name)]
            k[0] += ev.device_time_total / 1e3          # us -> ms
            k[1] += 1
    proofs = steps * batch
    step_ms = 1e3 * wall / proofs
    rows = sorted(({"kernel": n, "ms_per_proof": v[0] / proofs, "launches_per_proof": v[1] / proofs,
                    "share_of_step": v[0] / proofs / step_ms} for n, v in per.items()), key=lambda r: -r["ms_per_proof"])
    return {"step_ms_per_proof": step_ms, "kernel_ms_per_proof": sum(r["ms_per_proof"] for r in rows), "kernels": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2, help="profiled batches per lane setting (>= 1)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--top", type=int, default=40, help="kernels printed per lane setting")
    ap.add_argument("--json", metavar="OUT", help="also write the full breakdown as JSON")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    import torch
    import zkemail_b200 as z
    if not torch.cuda.is_available() or z.device_count() == 0:
        raise SystemExit("kernel_breakdown.py needs a CUDA device")
    circuit = z.Circuit(*bench.CIRCUIT)
    key = z.synthetic.generate_key(seed=bench.RSA_SEED)
    zk = z.Zkey(circuit, seed=bench.KEY_SEED, device=0)
    batch = bench.BATCH
    ctx = z.Context(circuit, zk, device=0, max_batch=batch)
    ctx.upload_inputs(b"".join(bench.make_inputs(z, circuit, batch, key)), batch)
    rs = bench.fixed_rs(batch)
    result = {"gpu": gpu_info(), "workload": "bench.py headline: %s%s, batch %d, domain 2^%d"
              % (bench.CIRCUIT[0], tuple(bench.CIRCUIT[1]), batch, circuit.info.domain_log2), "runs": {}}
    lanes_max = z._lib.zke_ctx_set_lanes(ctx.handle, 64)
    for lanes in (lanes_max, 1):
        z._lib.zke_ctx_set_lanes(ctx.handle, lanes)
        for _ in range(args.warmup):
            ctx.submit(None, batch, rs)
            ctx.collect()
        result["runs"]["lanes=%d" % lanes] = profile_run(torch, ctx, batch, rs, args.steps)
    result["gpu_after"] = gpu_info()
    ctx.close()

    print("# %s" % result["workload"])
    print("# gpu: %s" % json.dumps(result["gpu"]))
    print("# gpu after the runs: %s" % json.dumps(result["gpu_after"]))
    for label, run in result["runs"].items():
        print("\n## %s: step %.3f ms/proof (wall), kernels %.3f ms/proof (GPU time, summed)"
              % (label, run["step_ms_per_proof"], run["kernel_ms_per_proof"]))
        print("%10s %9s %7s  %s" % ("ms/proof", "launches", "share", "kernel"))
        for r in run["kernels"][: args.top]:
            print("%10.4f %9.2f %7.3f  %s" % (r["ms_per_proof"], r["launches_per_proof"], r["share_of_step"], r["kernel"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
