"""Cost of hashed and committed reveals (`"reveal": "hash" | "commit"`) and of the witness kernel's native Poseidon op, on
one GPU.

Two apps at the same sizes (default EmailVerifier(1024, 1536), compact regex shape): the commit app has a sender address
committed with a private salt (PoseidonModular then Poseidon(2)) and a hashed order id; the plain app reveals the same two
parts as bytes.  For each: proofs/s of Context.fullprove at batch 64 (host clock around synchronous calls, after one
warm-up batch; median of --repeats), the witness stage of a batch of 64 from the library's stage profile with
ZKE_NATIVE_POSEIDON=1 and =0 (read when a context opens), the single-email fullProve latency (a max_batch 1 context,
median of --repeats), and the program's levels with and without the op (the host lowering, cluster 1).  Every email is a
synthetic DKIM-signed one (zkemail_b200.synthetic, fixed key).  Prints one JSON object with the card's name, power limit
and SM clocks read by nvidia-smi in the same run.

    python scripts/commit_bench.py [--headers 1024] [--body 1536] [--batch 64] [--repeats 3] [--out FILE]
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


def app_spec(reveal: bool) -> dict:
    sender = {"regexDef": "[a-zA-Z0-9._%+-]+@[a-zA-Z0-9.-]+", "isPublic": True, "maxLength": 64}
    order = {"regexDef": "[0-9]+", "isPublic": True, "maxLength": 10}
    ext = [{"name": "recipient"}]
    if reveal:
        sender.update(reveal="commit", salt="senderSalt")
        order.update(reveal="hash")
        ext.append({"name": "senderSalt", "isPublic": False})
    return {
        "regexStyle": 1,
        "regexes": [
            {"name": "sender", "location": "header",
             "parts": [{"regexDef": "(\r\n|^)from:"}, {"regexDef": "([^\r\n]+<)?"}, sender, {"regexDef": ">?\r\n"}]},
            {"name": "order", "location": "body", "parts": [{"regexDef": "Order #"}, order]},
        ],
        "externalInputs": ext,
    }


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _inputs(spec, n):
    key = z.synthetic.generate_key(seed=77)
    rec = z.synthetic.key_record(key)
    out = []
    for i in range(n):
        em = z.synthetic.make_signed_email(i, key, body_len=1024, domain="gmail.com", marker=f"Order #{40000 + i} shipped")
        out.append(z.generate_app_inputs(em, spec, {"recipient": 7, "senderSalt": 1000 + i}, {"resolver": lambda nm, t: [rec]}))
    return out


def _median_time(fn, repeats):
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def bench(name, spec, batch, repeats):
    c = z.Circuit.from_spec(spec)
    inputs = _inputs(spec, min(batch, 8))
    packed = b"".join(c.pack_inputs(inputs[e % len(inputs)]) for e in range(batch))
    row = {"circuit": name, "constraints": c.info.n_constraints, "domain_log2": c.info.domain_log2,
           "levels_native_poseidon_1": c.program_stats()["n_levels"],
           "levels_native_poseidon_0": c.program_stats(native_poseidon=False)["n_levels"]}
    for flag in ("1", "0"):
        os.environ["ZKE_NATIVE_POSEIDON"] = flag
        cw = z.Context(c, None, device=0, max_batch=batch)
        cw.witness(packed, batch, want_witness=False)
        cw.profile(True)
        ms = []
        for _ in range(repeats):
            cw.witness(packed, batch, want_witness=False)
            ms.append(cw.profile_get()["witness"]["ms"])
        row["witness_ms_batch%d_native_poseidon_%s" % (batch, flag)] = round(statistics.median(ms[i] - (ms[i - 1] if i else 0) for i in range(len(ms))), 2)
        del cw
    os.environ.pop("ZKE_NATIVE_POSEIDON", None)
    zk = z.Zkey(c, seed=3)
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    ctx.fullprove(packed, batch)                                           # warm-up
    t = _median_time(lambda: ctx.fullprove(packed, batch), repeats)
    row["proofs_per_s_batch%d" % batch] = round(batch / t, 2)
    del ctx
    c1 = z.Context(c, zk, device=0, max_batch=1)
    one = c.pack_inputs(inputs[0])
    c1.fullprove(one, 1)
    row["fullprove_1_ms"] = round(1000 * _median_time(lambda: c1.fullprove(one, 1), repeats), 1)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--headers", type=int, default=1024)
    ap.add_argument("--body", type=int, default=1536)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    if z.device_count() == 0:
        raise SystemExit("commit_bench needs a CUDA device")
    sizes = {"maxHeadersLength": a.headers, "maxBodyLength": a.body}
    rows = []
    for name, reveal in (("commit app (hash + commit)", True), ("plain app (bytes)", False)):
        rows.append(bench(name, dict(app_spec(reveal), **sizes), a.batch, a.repeats))
        print(json.dumps(rows[-1]), flush=True)
    res = dict(_gpu_info(), headers=a.headers, body=a.body, batch=a.batch, repeats=a.repeats, regex_style=1, results=rows)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
