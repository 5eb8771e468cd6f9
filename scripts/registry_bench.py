"""Cost of the key registry on one GPU: batched Poseidon, the PoseidonLarge leaves and the Merkle tree, and what a hidden
key adds to an app.

- zke_poseidon_batch at widths 2 and 9 over 2^20 instances: hashes/s from the device time (CUDA events around the
  kernel, zke_registry_device_ms) and from the host-to-host wall time of the call (copies in and out included).
- zke_pubkey_hashes and zke_merkle_build (depth 20) at 2^10, 2^16 and 2^20 keys, device and host-to-host times.
- The 2^16 tree hashed by a single-threaded host loop over zke_poseidon_hash (the library's CPU permutation, one call per
  node, ctypes overhead included), labelled as such.
- The compact-shape hidden-sender app at EmailVerifier(1024, 1536) without and with "keyRegistryDepth": 20: constraints,
  domain, levels of the witness program, the witness stage of a batch of 64 (the library's stage profile) and proofs/s of
  Context.fullprove at batch 64 (host clock around synchronous calls, after one warm-up batch; median of --repeats).
- The derived arithmetic bound of the 2^20 leaves: ~7.6e9 field products at the 59.9 G products/s of
  profiles/field_peaks_h100.txt (~0.13 s), against the measured leaf time.
Prints one JSON object with the card's name, power limit and SM clocks read by nvidia-smi in the same run.

    python scripts/registry_bench.py [--repeats 3] [--out FILE]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "zk-email-verify_b200", "host")):
    if p not in sys.path:
        sys.path.insert(0, p)

import zkemail_b200 as z  # noqa: E402
from zkemail_b200 import _lib as L  # noqa: E402

R = z.FR_MODULUS
FIELD_PRODUCTS_PER_S = 59.9e9          # profiles/field_peaks_h100.txt


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _timed(fn, repeats):
    """(median host-to-host ms, median device ms) over `repeats` calls after one warm-up."""
    fn()
    host, dev = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        host.append(1e3 * (time.perf_counter() - t0))
        dev.append(L.zke_registry_device_ms())
    return statistics.median(host), statistics.median(dev)


def bench_batch(width, count, repeats):
    rng = random.Random(width)
    data = b"".join(rng.randrange(R).to_bytes(32, "little") for _ in range(width * count))
    out, err = ctypes.create_string_buffer(32 * count), ctypes.create_string_buffer(L.ERRCAP)

    def run():
        if L.zke_poseidon_batch(data, width, count, 0, out, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
    host, dev = _timed(run, repeats)
    return {"width": width, "count": count, "device_ms": round(dev, 3), "host_ms": round(host, 3),
            "hashes_per_s_device": round(count / (dev / 1e3)), "hashes_per_s_host_to_host": round(count / (host / 1e3))}


def bench_tree(m, depth, repeats):
    rng = random.Random(m)
    moduli = b"".join((rng.getrandbits(2048) | (1 << 2047) | 1).to_bytes(258, "little") for _ in range(m))
    leaves = ctypes.create_string_buffer(32 * m)
    err = ctypes.create_string_buffer(L.ERRCAP)

    def run_leaves():
        if L.zke_pubkey_hashes(moduli, m, 258, 121, 17, 0, leaves, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
    lh, ld = _timed(run_leaves, repeats)
    need = L.zke_merkle_build(leaves.raw, m, depth, 0, None, 0, err, L.ERRCAP)
    buf = ctypes.create_string_buffer(need)
    raw = leaves.raw

    def run_tree():
        if L.zke_merkle_build(raw, m, depth, 0, buf, need, err, L.ERRCAP) != need:
            raise L.ZkeError(err.value.decode())
    th, td = _timed(run_tree, repeats)
    return {"keys": m, "depth": depth, "leaves_device_ms": round(ld, 3), "leaves_host_ms": round(lh, 3),
            "tree_device_ms": round(td, 3), "tree_host_ms": round(th, 3), "tree_nodes": need // 32 - m}, raw, buf.raw


def host_loop_tree(raw_leaves, m, depth):
    """The same tree by one CPU thread calling zke_poseidon_hash per node."""
    level = [raw_leaves[32 * i:32 * i + 32] for i in range(m)]
    zero = bytes(32)
    out = ctypes.create_string_buffer(32)
    t0 = time.perf_counter()
    for _ in range(depth):
        nxt = []
        for j in range((len(level) + 1) // 2):
            right = level[2 * j + 1] if 2 * j + 1 < len(level) else zero
            if L.zke_poseidon_hash(level[2 * j] + right, 2, out) != 0:
                raise L.ZkeError("zke_poseidon_hash failed")
            nxt.append(out.raw)
        level = nxt
        zz = ctypes.create_string_buffer(32)
        L.zke_poseidon_hash(zero + zero, 2, zz)
        zero = zz.raw
    return 1e3 * (time.perf_counter() - t0), level[0]


def app_spec(depth):
    spec = {
        "regexStyle": 1,
        "regexes": [{"name": "sender", "location": "header",
                     "parts": [{"regexDef": "(\r\n|^)from:"}, {"regexDef": "([^\r\n]+<)?"},
                               {"regexDef": "[a-zA-Z0-9._%+-]+@[a-zA-Z0-9.-]+", "isPublic": True, "maxLength": 64,
                                "reveal": "commit", "salt": "senderSalt"}, {"regexDef": ">?\r\n"}]}],
        "externalInputs": [{"name": "senderSalt", "isPublic": False}],
    }
    if depth:
        spec["keyRegistryDepth"] = depth
    return spec


def bench_app(depth, batch, repeats):
    spec = app_spec(depth)
    c = z.Circuit.from_spec(spec)
    key = z.synthetic.generate_key(seed=77)
    rec = z.synthetic.key_record(key)
    params = {}
    if depth:
        rng = random.Random(3)
        keys = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(1 << 16)]
        keys[12345] = rec
        params["registry"] = z.KeyRegistry.build(keys, depth)
    packed = []
    for i in range(batch):
        em = z.synthetic.make_signed_email(i, key, domain="gmail.com")
        dk = z.verify_dkim_signature(em, resolver=lambda n, t: [rec])
        packed.append(c.pack_inputs(z.generate_app_inputs(dk, spec, {"senderSalt": 1000 + i}, params=dict(params))))
    data = b"".join(packed)
    cw = z.Context(c, None, device=0, max_batch=batch)
    cw.witness(data, batch, want_witness=False)
    cw.profile(True)
    wit = []
    for _ in range(repeats):                      # the stage profile accumulates: take the increments
        cw.witness(data, batch, want_witness=False)
        wit.append(cw.profile_get()["witness"]["ms"])
    wit = [wit[i] - (wit[i - 1] if i else 0) for i in range(len(wit))]
    del cw
    zk = z.Zkey(c, seed=7, device=0)
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    ctx.fullprove(data, batch)
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        ctx.fullprove(data, batch)
        times.append(time.perf_counter() - t0)
    st = c.program_stats()
    return {"keyRegistryDepth": depth, "constraints": c.info.n_constraints, "domain_log2": c.info.domain_log2,
            "levels": st["n_levels"], "witness_ms_batch": round(statistics.median(wit), 2),
            "batch": batch, "proofs_per_s": round(batch / statistics.median(times), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("registry_bench needs a CUDA device")
    res = {"card": _gpu_info()}
    res["poseidon_batch"] = [bench_batch(w, 1 << 20, a.repeats) for w in (2, 9)]
    trees = []
    for lg in (10, 16, 20):
        row, raw, levels = bench_tree(1 << lg, 20, a.repeats)
        if lg == 16:
            ms, root = host_loop_tree(raw, 1 << 16, 20)
            assert root == levels[-32:], "host loop and GPU tree disagree"
            res["host_loop_tree_2^16"] = {"label": "single-threaded host loop over zke_poseidon_hash, one call per node",
                                          "ms": round(ms, 1)}
        trees.append(row)
    res["trees"] = trees
    leaves_ms = trees[-1]["leaves_device_ms"]
    res["leaves_2^20_bound"] = {"field_products": 7.6e9, "derived_ms_at_59.9G_per_s": round(7.6e9 / FIELD_PRODUCTS_PER_S * 1e3, 1),
                                "measured_device_ms": leaves_ms}
    res["app"] = [bench_app(d, a.batch, a.repeats) for d in (0, 20)]
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
