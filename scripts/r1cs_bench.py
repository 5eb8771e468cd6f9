"""Time of circom's `.r1cs` route on one GPU (zk-email-verify_b200/csrc/r1cs.cpp, setup.cu, engine.cu) at the benchmark's
circuit.

Steps, each a synchronous library call timed by the host clock (every call that touches the device ends in a device
synchronisation):
  * the circuit exported natively as `.r1cs` (Circuit.write_r1cs) and read back (Circuit.from_r1cs, from memory);
  * Zkey.from_ptau on one toy `.ptau` of power domain_log2 + 1 for the template circuit and for the circuit read from its
    `.r1cs`, alternating, with the library's split into the host part (parse, transpose) and the device part (uploads, point
    validation, the signal sums, the H fixed-base table);
  * the same for a circom-shaped synthetic R1CS of the same domain and a similar term count, drawn like the generator of
    tests/test_r1cs_reader.py: every term's coefficient is 1, r - 1, 2^k, r - 2^k, a small constant or a full-width random
    value with equal odds, every third row linear.  The device part is reported per R1CS term for both;
  * Context.check_witness (`snarkjs wtns check`) of 64 witnesses loaded into a context on the `.r1cs` circuit, and the
    template context's own check of the same witnesses.
Prints one JSON line with the card's name, power limit and SM clock read by nvidia-smi in the same run.

    python scripts/r1cs_bench.py [--params 1024,1536,121,17] [--repeats 3] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import statistics
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "zk-email-verify_b200", "host")):
    if p not in sys.path:
        sys.path.insert(0, p)

import zkemail_b200 as z  # noqa: E402
from zkemail_b200 import _lib as L  # noqa: E402

R = z.FR_MODULUS


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t0


def _words(v: int) -> np.ndarray:
    return np.frombuffer(int(v).to_bytes(32, "little"), dtype="<u4")


def synthetic_r1cs(n_constraints: int, seed: int = 7) -> bytes:
    """A circom-shaped `.r1cs` with n_constraints rows: quadratic rows with 1-4 / 1-3 / 1-4 terms in A / B / C, every third
    row linear (A = B = 0, 1-4 terms in C), about one wire per row, coefficients drawn from six classes with equal odds."""
    rng = np.random.default_rng(seed)
    n_out, n_pub, n_prv = 2, 3, 4
    n_wires = n_constraints + 1 + n_out + n_pub + n_prv
    quad = (np.arange(n_constraints) % 3) != 2
    counts = np.zeros((n_constraints, 3), dtype=np.int64)
    counts[:, 0] = np.where(quad, rng.integers(1, 5, n_constraints), 0)
    counts[:, 1] = np.where(quad, rng.integers(1, 4, n_constraints), 0)
    counts[:, 2] = rng.integers(1, 5, n_constraints)
    counts = counts.ravel()
    nnz = int(counts.sum())
    wires = rng.integers(0, n_wires, nnz, dtype=np.uint32)
    cls = rng.integers(0, 6, nnz)
    k = rng.integers(1, 253, nnz)
    coef = np.zeros((nnz, 8), dtype="<u4")
    coef[cls == 0, 0] = 1
    coef[cls == 1] = _words(R - 1)
    sel = cls == 2
    coef[sel, k[sel] // 32] = (np.uint64(1) << (k[sel] % 32).astype(np.uint64)).astype("<u4")
    neg_pow2 = np.stack([_words(R - (1 << j)) if j else np.zeros(8, "<u4") for j in range(253)])
    coef[cls == 3] = neg_pow2[k[cls == 3]]
    sel = cls == 4
    coef[sel, 0] = rng.integers(2, 100, int(sel.sum()))
    sel = cls == 5
    full = rng.integers(0, 1 << 32, (int(sel.sum()), 8), dtype=np.uint64).astype("<u4")
    full[:, 7] %= int(_words(R)[7])          # below r: the top word is below r's
    coef[sel] = full
    terms = np.empty((nnz, 9), dtype="<u4")
    terms[:, 0] = wires
    terms[:, 1:] = coef
    total = counts.size + 9 * nnz
    words = np.empty(total, dtype="<u4")
    hdr = np.concatenate(([0], np.cumsum(1 + 9 * counts)[:-1]))
    mask = np.ones(total, dtype=bool)
    mask[hdr] = False
    words[hdr] = counts
    words[mask] = terms.ravel()
    del terms, mask
    header = struct.pack("<I", 32) + R.to_bytes(32, "little") + struct.pack("<IIIIQI", n_wires, n_out, n_pub, n_prv, n_wires, n_constraints)
    body = words.tobytes()
    labels = np.arange(n_wires, dtype="<u8").tobytes()
    out = bytearray(b"r1cs" + struct.pack("<II", 1, 3))
    for typ, payload in ((1, header), (2, body), (3, labels)):
        out += struct.pack("<IQ", typ, len(payload)) + payload
    return bytes(out)


def from_ptau_split(c, ptau):
    key, t = _timed(lambda: z.Zkey.from_ptau(c, ptau))
    host_ms, gpu_ms = ctypes.c_double(), ctypes.c_double()
    L.zke_zkey_from_ptau_timing(ctypes.byref(host_ms), ctypes.byref(gpu_ms))
    del key
    return t, host_ms.value / 1e3, gpu_ms.value / 1e3


def _med(xs):
    return round(statistics.median(xs), 3)


def _resolver(k):
    return lambda n, t: [z.synthetic.key_record(k)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", default="1024,1536,121,17")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("r1cs_bench needs a CUDA device")
    params = [int(v) for v in args.params.split(",") if v]
    c = z.Circuit("EmailVerifier", params)
    i = c.info
    res = {"circuit": f"EmailVerifier({args.params})", "n_vars": i.n_vars, "n_constraints": i.n_constraints,
           "domain_log2": i.domain_log2, "terms": i.nnz_a + i.nnz_b + i.nnz_c, "ptau_power": i.domain_log2 + 1}
    # warm-up: module load and device set-up on a small circuit, both routes
    small = z.Circuit("SelectRegexReveal", [34, 8])
    z.Zkey.from_ptau(z.Circuit.from_r1cs(small.write_r1cs()), z.ptau_toy(11, 3, 5, 7))

    blob, t = _timed(c.write_r1cs)
    res["write_r1cs_s"], res["r1cs_bytes"] = round(t, 3), len(blob)
    rc, t = _timed(lambda: z.Circuit.from_r1cs(blob))
    res["from_r1cs_s"] = round(t, 3)
    del blob

    syn_rows = (1 << (i.domain_log2 - 1)) + (1 << (i.domain_log2 - 4))     # the same domain as the template circuit
    sblob, t = _timed(lambda: synthetic_r1cs(syn_rows))
    syn, t = _timed(lambda: z.Circuit.from_r1cs(sblob))
    si = syn.info
    assert si.domain_log2 == i.domain_log2
    res["synthetic"] = {"n_constraints": si.n_constraints, "terms": si.nnz_a + si.nnz_b + si.nnz_c, "r1cs_bytes": len(sblob),
                        "from_r1cs_s": round(t, 3)}
    del sblob

    ptau, t = _timed(lambda: z.ptau_toy(i.domain_log2 + 1, 0x1234567 * 10 ** 40 + 1, 0xABCDEF, 0x13579))
    res["ptau_toy_s"], res["ptau_bytes"] = round(t, 3), len(ptau)
    runs = {"template": [], "r1cs": [], "synthetic": []}
    for _ in range(args.repeats):
        for name, circ in (("template", c), ("r1cs", rc), ("synthetic", syn)):
            runs[name].append(from_ptau_split(circ, ptau))
    del ptau
    for name, rr in runs.items():
        total, host, gpu = (_med([r[j] for r in rr]) for j in range(3))
        terms = res["terms"] if name != "synthetic" else res["synthetic"]["terms"]
        res["from_ptau_" + name] = {"total_s": total, "host_s": host, "gpu_s": gpu,
                                    "gpu_ns_per_term": round(1e9 * statistics.median([r[2] for r in rr]) / terms, 2)}
    res["synthetic_over_template_per_term"] = round(res["from_ptau_synthetic"]["gpu_ns_per_term"] /
                                                    res["from_ptau_template"]["gpu_ns_per_term"], 2)
    del syn

    # wtns check: witnesses from the template circuit's own witness program, loaded into a context on the `.r1cs` circuit
    b = args.batch
    k = z.synthetic.generate_key(seed=5)
    emails = []
    for j in range(4):
        dk = z.verify_dkim_signature(z.synthetic.make_signed_email(40 + j, k, body_len=params[1] // 2), resolver=_resolver(k))
        emails.append(c.pack_inputs(z.generate_email_verifier_inputs_from_dkim_result(
            dk, {"maxHeadersLength": params[0], "maxBodyLength": params[1]})))
    ctx_t = z.Context(c, device=0, max_batch=b)
    wt, status = ctx_t.witness(b"".join(emails[j % 4] for j in range(b)), b)
    assert status == [-1] * b
    ctx_r = z.Context(rc, device=0, max_batch=b)
    _, t = _timed(lambda: ctx_r.load_witness(wt, b))
    res["check_witness"] = {"batch": b, "load_witness_s": round(t, 3)}
    ctx_t.load_witness(wt, b)
    del wt
    for name, ctx in (("r1cs", ctx_r), ("template", ctx_t)):
        assert ctx.check_witness(b) == [-1] * b     # warm-up
        times = [_timed(lambda: ctx.check_witness(b))[1] for _ in range(5)]
        res["check_witness"][name + "_ms"] = round(1e3 * statistics.median(times), 2)
    ctx_t.close()
    ctx_r.close()
    res.update(_gpu_info())
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
