"""Time of phase 1 of the Powers-of-Tau ceremony on one GPU (zk-email-verify_b200/csrc/ptau.cu) at one power.

Steps, each a synchronous library call timed by the host clock (every call ends in a device synchronisation):
  * ptau_new (host only);
  * ptau_contribute on the new file (every point times its own scalar);
  * ptau_prepare of the contributed file, with its split into the three G1 families and the G2 family as the library
    measured it;
  * verify_ptau on the unprepared and on the prepared file, and on the prepared file with the previous file and the receipt.
The prepared file is asserted equal, byte for byte, to ptau_toy at the same secrets.  Twiddle multiplications per second
count the transform's variable-base multiplications: for the domains 2^0 .. 2^power, sum_k k 2^(k-1) = (power - 1) 2^power + 1
per family (the j = 0 butterflies, which skip the multiplication, are included).  Prints one JSON line with the card's name,
power limit and SM clocks read by nvidia-smi in the same run.

    python scripts/ptau_bench.py [--power 23] [--out FILE]
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

SECRETS = (0x1234567 * 10 ** 40 + 1, 0xABCDEF, 0x13579)


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
    ap.add_argument("--power", type=int, default=23)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("ptau_bench needs a CUDA device")
    p = args.power
    twiddles = (p - 1) * (1 << p) + 1
    res = {"power": p, "twiddle_muls_per_family": twiddles}
    # warm-up: module load and device set-up at a small power
    small, rc = z.ptau_contribute(z.ptau_new(6), SECRETS)
    z.verify_ptau(z.ptau_prepare(small), prev=z.ptau_new(6), receipt=rc)

    new, t = _timed(lambda: z.ptau_new(p))
    res["new_s"] = round(t, 3)
    (c1, receipt), t = _timed(lambda: z.ptau_contribute(new, SECRETS))
    res["contribute_s"] = round(t, 3)
    prep, t = _timed(lambda: z.ptau_prepare(c1))
    g1_ms, g2_ms = ctypes.c_double(), ctypes.c_double()
    L.zke_ptau_prepare_timing(ctypes.byref(g1_ms), ctypes.byref(g2_ms))
    res["prepare_s"] = round(t, 3)
    res["prepare_g1_s"], res["prepare_g2_s"] = round(g1_ms.value / 1e3, 3), round(g2_ms.value / 1e3, 3)
    res["g1_twiddle_muls_per_s"] = round(3 * twiddles / (g1_ms.value / 1e3))
    res["g2_twiddle_muls_per_s"] = round(twiddles / (g2_ms.value / 1e3))
    res["prepared_bytes"] = len(prep)
    toy = z.ptau_toy(p, *SECRETS)
    assert prep == toy, "the prepared file differs from ptau_toy at the same secrets"
    res["prepared_equals_ptau_toy"] = True
    del toy
    rand = bytes(range(16))
    ok, t = _timed(lambda: z.verify_ptau(c1, rand=rand))
    assert ok
    res["verify_unprepared_s"] = round(t, 3)
    ok, t = _timed(lambda: z.verify_ptau(prep, rand=rand))
    assert ok
    res["verify_prepared_s"] = round(t, 3)
    ok, t = _timed(lambda: z.verify_ptau(prep, prev=new, receipt=receipt, rand=rand))
    assert ok
    res["verify_prepared_with_prev_s"] = round(t, 3)
    res.update(_gpu_info())
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
