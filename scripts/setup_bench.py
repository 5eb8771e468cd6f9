"""Time of the Powers-of-Tau key route on one GPU (zk-email-verify_b200/csrc/setup.cu) at the benchmark's circuit.

Steps, each a synchronous library call timed by the host clock (every call ends in a device synchronisation):
  * toy `.ptau` generation (zke_ptau_toy) for power domain_log2 + 1 - reported, but only a stand-in for a ceremony file;
  * Zkey.from_ptau, with its split into the host part (parse, transpose to signal-major terms) and the device part
    (uploads, point validation, the signal sums, the H fixed-base table) as the library measured it;
  * Zkey.contribute (C and H times one scalar, the H table rebuilt);
  * Zkey.check_contribution (two G1 multi-exponentiations per key and the pairings).
Prints one JSON line with the card's name, power limit and SM clock read by nvidia-smi in the same run.

    python scripts/setup_bench.py [--template EmailVerifier --params 1024,1536,121,17] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "zk-email-verify_b200", "host")):
    if p not in sys.path:
        sys.path.insert(0, p)

import zkemail_b200 as z  # noqa: E402
from zkemail_b200 import _lib as L  # noqa: E402


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--template", default="EmailVerifier")
    ap.add_argument("--params", default="1024,1536,121,17")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("setup_bench needs a CUDA device")
    params = [int(v) for v in args.params.split(",") if v]
    c = z.Circuit(args.template, params)
    i = c.info
    res = {"circuit": f"{args.template}({args.params})", "n_vars": i.n_vars, "n_public": i.n_public, "domain_log2": i.domain_log2,
           "nnz_a": i.nnz_a, "nnz_b": i.nnz_b, "nnz_c": i.nnz_c, "ptau_power": i.domain_log2 + 1}
    # warm-up: module load and device set-up on a small circuit
    small = z.Circuit("SelectRegexReveal", [34, 8])
    z.Zkey.from_ptau(small, z.ptau_toy(11, 3, 5, 7)).contribute(b"\x02" + bytes(31))

    ptau, t = _timed(lambda: z.ptau_toy(i.domain_log2 + 1, 0x1234567 * 10 ** 40 + 1, 0xABCDEF, 0x13579))
    res["ptau_toy_s"], res["ptau_bytes"] = round(t, 3), len(ptau)
    base, t = _timed(lambda: z.Zkey.from_ptau(c, ptau))
    host_ms, gpu_ms = ctypes.c_double(), ctypes.c_double()
    L.zke_zkey_from_ptau_timing(ctypes.byref(host_ms), ctypes.byref(gpu_ms))
    res["from_ptau_s"] = round(t, 3)
    res["from_ptau_host_s"], res["from_ptau_gpu_s"] = round(host_ms.value / 1e3, 3), round(gpu_ms.value / 1e3, 3)
    del ptau
    key, t = _timed(lambda: base.contribute((0x5EC2E7 * 10 ** 30 + 17).to_bytes(32, "little")))
    res["contribute_s"] = round(t, 3)
    ok, t = _timed(lambda: key.check_contribution(base, bytes(range(16))))
    assert ok, "an honest contribution was rejected"
    res["check_contribution_s"] = round(t, 3)
    res.update(_gpu_info())
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
