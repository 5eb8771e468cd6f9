"""Cost of domain-bound registry leaves on one GPU, and what binding the leaf to a domain adds to an app.

- zke_domain_key_leaves at 2^10, 2^16 and 2^20 (domain, key) pairs beside zke_pubkey_hashes on the same moduli: device
  time (CUDA events around the kernel, zke_registry_device_ms) and host-to-host wall time of the call (copies included),
  medians of --repeats after one warm-up.
- The compact-shape app of scripts/registry_bench.py at EmailVerifier(1024, 1536) with "keyRegistryDepth": 20 and a
  public `d=` tag part, without and with "keyDomain" on that part: constraints, domain, levels of the witness program,
  the witness stage of a batch of 64 (the library's stage profile) and proofs/s of Context.fullprove at batch 64.
Prints one JSON object with the card's name, power limit and SM clocks read by nvidia-smi in the same run.

    python scripts/domain_registry_bench.py [--repeats 3] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from registry_bench import _gpu_info, _timed, app_spec  # noqa: E402
import zkemail_b200 as z  # noqa: E402
from zkemail_b200 import _lib as L  # noqa: E402

MBYTES = 258                            # n k = 2057 bits


def bench_leaves(m, repeats):
    rng = random.Random(m)
    moduli = b"".join((rng.getrandbits(2048) | (1 << 2047) | 1).to_bytes(MBYTES, "little") for _ in range(m))
    rows = b"".join(f"mail{i}.example{i % 97}.com".encode().ljust(255, b"\0") for i in range(m))
    out, err = ctypes.create_string_buffer(32 * m), ctypes.create_string_buffer(L.ERRCAP)

    def run_domain():
        if L.zke_domain_key_leaves(moduli, m, MBYTES, 121, 17, rows, 0, out, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())

    def run_plain():
        if L.zke_pubkey_hashes(moduli, m, MBYTES, 121, 17, 0, out, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
    dh, dd = _timed(run_domain, repeats)
    ph, pd = _timed(run_plain, repeats)
    return {"pairs": m, "domain_key_leaves_device_ms": round(dd, 3), "domain_key_leaves_host_ms": round(dh, 3),
            "pubkey_hashes_device_ms": round(pd, 3), "pubkey_hashes_host_ms": round(ph, 3)}


def domain_app_spec(bound):
    spec = app_spec(20)
    spec["regexes"].append({"name": "dkimDomain", "location": "header",
                            "parts": [{"regexDef": "(\r\n|^)dkim-signature:"}, {"regexDef": "([a-z]+=[^;]+; )+d="},
                                      {"regexDef": "[a-z0-9.-]+", "isPublic": True, "maxLength": 64}, {"regexDef": ";"}]})
    if bound:
        spec["keyDomain"] = "dkimDomain"
    return spec


def bench_app(bound, batch, repeats):
    spec = domain_app_spec(bound)
    c = z.Circuit.from_spec(spec)
    key = z.synthetic.generate_key(seed=77)
    rec = z.synthetic.key_record(key)
    rng = random.Random(3)
    keys = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(1 << 16)]
    keys[12345] = rec
    if bound:
        reg = z.KeyRegistry.build_domains([(f"mail{i}.example.com", x) if i != 12345 else ("gmail.com", x)
                                           for i, x in enumerate(keys)], 20)
    else:
        reg = z.KeyRegistry.build(keys, 20)
    packed = []
    for i in range(batch):
        em = z.synthetic.make_signed_email(i, key, domain="gmail.com")
        dk = z.verify_dkim_signature(em, resolver=lambda n, t: [rec])
        packed.append(c.pack_inputs(z.generate_app_inputs(dk, spec, {"senderSalt": 1000 + i}, params={"registry": reg})))
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
    return {"keyDomain": spec.get("keyDomain"), "keyRegistryDepth": 20, "constraints": c.info.n_constraints,
            "domain_log2": c.info.domain_log2, "levels": st["n_levels"], "witness_ms_batch": round(statistics.median(wit), 2),
            "batch": batch, "proofs_per_s": round(batch / statistics.median(times), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("domain_registry_bench needs a CUDA device")
    res = {"card": _gpu_info()}
    res["leaves"] = [bench_leaves(1 << lg, a.repeats) for lg in (10, 16, 20)]
    res["app"] = [bench_app(b, a.batch, a.repeats) for b in (False, True)]
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
