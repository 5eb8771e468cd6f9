"""Cost of updating a key registry in place on one GPU, against rebuilding it.

Setup: a depth-20 registry of 2^20 random leaves, resident on the device (zke_registry_open, itself timed).
- zke_registry_update with k = 1, 64, 4,096 and 65,536 random distinct replacements (the same k pairs in every call), and
  an append of 4,096 leaves to a registry of 2^20 - 4,096 (repeats + 1) leaves (each call appends the next 4,096; the
  warm-up call also doubles the capacity, reported on its own).
- zke_registry_nodes for 64 full authentication paths (64 x 20 nodes).
- KeyRegistry.update of 64 leaves host to host, the patching of KeyRegistry.levels included.
- Baselines on the final leaves of the replacements: zke_merkle_build (device and host to host) and
  KeyRegistry.from_leaves (host to host: the build plus turning ~2.1 M nodes into Python ints).  The resident levels
  are checked equal to zke_merkle_build's byte for byte.
Each update reports the node hashes it performed, counted here from its indices (the distinct ancestors idx >> l at
levels 1..20), and hashes/s from the device and from the host-to-host times.  Device time is zke_registry_device_ms (CUDA
events around the call's kernels), host-to-host the wall time around the call; medians of --repeats calls after one
warm-up.  Prints one JSON object with the card's name, power limit and SM clocks read by nvidia-smi in the same run.

    python scripts/registry_update_bench.py [--repeats 5] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import subprocess
import sys
import time
from array import array

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "zk-email-verify_b200", "host")):
    if p not in sys.path:
        sys.path.insert(0, p)

import zkemail_b200 as z  # noqa: E402
from zkemail_b200 import _lib as L  # noqa: E402

R = z.FR_MODULUS
DEPTH = 20
M = 1 << DEPTH


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _call(fn):
    t0 = time.perf_counter()
    fn()
    return 1e3 * (time.perf_counter() - t0), L.zke_registry_device_ms()


def _timed(fn, repeats):
    """(median host-to-host ms, median device ms) over `repeats` calls after one warm-up."""
    fn()
    runs = [_call(fn) for _ in range(repeats)]
    return statistics.median(h for h, _ in runs), statistics.median(d for _, d in runs)


def _hashes(indices):
    """Node hashes of an update of these leaf indices: the distinct ancestors at levels 1..DEPTH."""
    n, cur = 0, set(indices)
    for _ in range(DEPTH):
        cur = {i >> 1 for i in cur}
        n += len(cur)
    return n


def _image(leaves):
    return b"".join(x.to_bytes(32, "little") for x in leaves)


def _open(leaves):
    err = ctypes.create_string_buffer(L.ERRCAP)
    h = L.zke_registry_open(_image(leaves), len(leaves), DEPTH, 0, err, L.ERRCAP)
    if not h:
        raise L.ZkeError(err.value.decode())
    return h


def _update(h, indices, leaves):
    idx, data, err = array("Q", indices).tobytes(), _image(leaves), ctypes.create_string_buffer(L.ERRCAP)

    def run():
        if L.zke_registry_update(h, idx, data, len(indices), err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
    return run


def _row(name, k, hashes, host, dev):
    return {"workload": name, "k": k, "node_hashes": hashes, "device_ms": round(dev, 4), "host_ms": round(host, 4),
            "hashes_per_s_device": round(hashes / (dev / 1e3)), "hashes_per_s_host_to_host": round(hashes / (host / 1e3))}


def _levels(h):
    err = ctypes.create_string_buffer(L.ERRCAP)
    need = L.zke_registry_levels(h, None, 0, err, L.ERRCAP)
    buf = ctypes.create_string_buffer(need)
    if L.zke_registry_levels(h, buf, need, err, L.ERRCAP) != need:
        raise L.ZkeError(err.value.decode())
    return buf.raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.repeats < 3:
        raise SystemExit("--repeats must be at least 3")
    if z.device_count() == 0:
        raise SystemExit("registry_update_bench needs a CUDA device")
    res = {"card": _gpu_info(), "depth": DEPTH, "leaves": M, "repeats": a.repeats}
    rng = random.Random(20)
    leaves = [rng.randrange(R) for _ in range(M)]

    host, dev = _timed(lambda: L.zke_registry_close(_open(leaves)), a.repeats)
    res["open"] = {"device_ms": round(dev, 3), "host_ms": round(host, 3)}
    h = _open(leaves)
    rows = []
    for k in (1, 64, 4096, 65536):
        idx = rng.sample(range(M), k)
        new = [rng.randrange(R) for _ in range(k)]
        host, dev = _timed(_update(h, idx, new), a.repeats)
        for i, x in zip(idx, new):
            leaves[i] = x
        rows.append(_row("replace", k, _hashes(idx), host, dev))

    # paths of 64 leaves: levels 0..19, the sibling of the ancestor at each
    picks = rng.sample(range(M), 64)
    lv = array("I", [l for _ in picks for l in range(DEPTH)]).tobytes()
    ix = array("Q", [(i >> l) ^ 1 for i in picks for l in range(DEPTH)]).tobytes()
    out, err = ctypes.create_string_buffer(32 * 64 * DEPTH), ctypes.create_string_buffer(L.ERRCAP)

    def paths():
        if L.zke_registry_nodes(h, lv, ix, 64 * DEPTH, out, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
    host, dev = _timed(paths, a.repeats)
    res["nodes_64_paths"] = {"nodes": 64 * DEPTH, "device_ms": round(dev, 4), "host_ms": round(host, 4)}

    # baselines on the final leaves; the resident tree must equal the rebuild
    data = _image(leaves)
    need = L.zke_merkle_build(data, M, DEPTH, 0, None, 0, err, L.ERRCAP)
    buf = ctypes.create_string_buffer(need)

    def rebuild():
        if L.zke_merkle_build(data, M, DEPTH, 0, buf, need, err, L.ERRCAP) != need:
            raise L.ZkeError(err.value.decode())
    host, dev = _timed(rebuild, a.repeats)
    res["merkle_build"] = {"node_hashes": M - 1, "device_ms": round(dev, 3), "host_ms": round(host, 3)}
    assert _levels(h) == buf.raw, "resident levels differ from zke_merkle_build"
    host, dev = _timed(lambda: _levels(h), a.repeats)
    res["registry_levels_copy"] = {"device_ms": round(dev, 3), "host_ms": round(host, 3)}
    L.zke_registry_close(h)

    # append: 4,096 leaves per call into room for warm-up + repeats calls
    k = 4096
    start = M - k * (a.repeats + 1)
    h = _open(leaves[:start])
    calls = []
    for c in range(a.repeats + 1):
        idx = list(range(start + c * k, start + (c + 1) * k))
        host, dev = _call(_update(h, idx, leaves[start + c * k:start + (c + 1) * k]))
        calls.append((host, dev, _hashes(idx)))
    res["append_first_call_with_growth"] = {"k": k, "device_ms": round(calls[0][1], 4), "host_ms": round(calls[0][0], 4)}
    rows.append(_row("append", k, statistics.median(c[2] for c in calls[1:]), statistics.median(c[0] for c in calls[1:]),
                     statistics.median(c[1] for c in calls[1:])))
    assert _levels(h) == buf.raw, "resident levels after appends differ from zke_merkle_build"
    L.zke_registry_close(h)
    res["update"] = rows

    # KeyRegistry: rebuild from scratch against an update of 64 leaves with its mirror
    times = []
    for _ in range(a.repeats + 1):
        t0 = time.perf_counter()
        reg = z.KeyRegistry.from_leaves(leaves, DEPTH)
        times.append(1e3 * (time.perf_counter() - t0))
    res["keyregistry_from_leaves_host_ms"] = round(statistics.median(times[1:]), 3)
    idx = rng.sample(range(M), 64)
    changes = [{i: rng.randrange(R) for i in idx} for _ in range(a.repeats + 1)]
    reg.update(changes[0])                           # opens the resident tree
    times = []
    for ch in changes[1:]:
        t0 = time.perf_counter()
        reg.update(ch)
        times.append(1e3 * (time.perf_counter() - t0))
    hashes = _hashes(idx)
    host = statistics.median(times)
    res["keyregistry_update_64"] = {"node_hashes": hashes, "host_ms": round(host, 4),
                                    "hashes_per_s_host_to_host": round(hashes / (host / 1e3))}
    assert reg.root == z.registry.merkle_levels(reg.leaves, DEPTH)[-1][0]
    reg.close()

    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
