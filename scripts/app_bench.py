"""Throughput of email app circuits (Circuit.from_spec) on one GPU, beside TwitterVerifier at the same sizes.

For each circuit: proofs/s of Context.fullprove at batch 64 (witness kernel + proof, host clock around synchronous calls,
after one warm-up batch; median of --repeats), the single-email fullProve latency (a max_batch 1 context, median of
--repeats), and the circuit's constraint count and domain.  For the app in both regex shapes, the witness stage of a batch
of 64 with regex seeding on (ZKE_NATIVE_REGEX=1) and off (=0), from the library's stage profile.  Every email is a
synthetic DKIM-signed one (zkemail_b200.synthetic, fixed key).  Prints one JSON object with the card's name, power limit
and SM clocks read by nvidia-smi in the same run.

    python scripts/app_bench.py [--headers 1024] [--body 1536] [--batch 64] [--repeats 3] [--out FILE]
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

# Proof-of-Twitter as a spec: TwitterVerifier's circuit exactly (tests/test_app_circuit.py checks the identity)
TWITTER_SPEC = {
    "maxHeadersLength": 1024, "maxBodyLength": 1536, "n": 121, "k": 17, "exposeHeaderHash": False,
    "regexes": [{"name": "twitterUsername", "location": "body",
                 "parts": [{"regexDef": "email was meant for @"},
                           {"regexDef": "[a-zA-Z0-9_]+", "isPublic": True, "maxLength": 21}]}],
    "externalInputs": [{"name": "address"}],
}
RECIPIENT = "0x71C7656EC7ab88b098defB751B7401B5f6d8976F"
SUBJECT = "Your order of 3 books"


def app_spec(style: int) -> dict:
    """The multi-regex app of tests/test_app_circuit.py: header from-address, the subject line, a body regex with two
    public parts, the sender-domain regex (74 DFA states: the wide seeding mode), a string external input, the nullifier."""
    return {
        "maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": style,
        "regexes": [
            {"name": "fromAddress", "location": "header",
             "parts": [{"regexDef": "(\r\n|^)from:"}, {"regexDef": "([^\r\n]+<)?"},
                       {"regexDef": "[a-zA-Z0-9._%+-]+@[a-zA-Z0-9.-]+", "isPublic": True, "maxLength": 64},
                       {"regexDef": ">?\r\n"}]},
            {"name": "subject", "location": "header",
             "parts": [{"regexDef": "(\r\n|^)subject:"}, {"regexDef": "[^\r\n]+", "isPublic": True, "maxLength": 64},
                       {"regexDef": "\r\n"}]},
            {"name": "order", "location": "body",
             "parts": [{"regexDef": "Order #"}, {"regexDef": "[0-9]+", "isPublic": True, "maxLength": 10},
                       {"regexDef": " shipped to "}, {"regexDef": "[A-Za-z]+", "isPublic": True, "maxLength": 20}]},
            {"name": "senderDomain", "location": "header",
             "parts": [{"regexDef": "from:[^\r\n]*@"},
                       {"regexDef": "(gmail\\.com|icloud\\.com|outlook\\.com|yahoo\\.com|proton\\.me)", "isPublic": True, "maxLength": 31}]},
        ],
        "externalInputs": [{"name": "recipient", "maxLength": 42}],
        "emailNullifier": True,
    }


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _inputs(spec, n, twitter):
    key = z.synthetic.generate_key(seed=77)
    rec = z.synthetic.key_record(key)
    out = []
    for i in range(n):
        marker = f"This email was meant for @user{i}" if twitter else f"Order #{40000 + i} shipped to Carol"
        em = z.synthetic.make_signed_email(i, key, body_len=1024, domain="gmail.com", marker=marker, subject=SUBJECT)
        ext = {"address": 0x1234} if twitter else {"recipient": RECIPIENT}
        out.append(z.generate_app_inputs(em, spec, ext, {"resolver": lambda nm, t: [rec]}))
    return out


def _median_time(fn, repeats):
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def bench(name, spec, batch, repeats, twitter=False, seeding_ab=False):
    c = z.Circuit.from_spec(spec)
    inputs = _inputs(spec, min(batch, 8), twitter)
    packed = b"".join(c.pack_inputs(inputs[e % len(inputs)]) for e in range(batch))
    zk = z.Zkey(c, seed=3)
    row = {"circuit": name, "constraints": c.info.n_constraints, "domain_log2": c.info.domain_log2}
    ctx = z.Context(c, zk, device=0, max_batch=batch)
    ctx.fullprove(packed, batch)                                           # warm-up
    t = _median_time(lambda: ctx.fullprove(packed, batch), repeats)
    row["proofs_per_s_batch%d" % batch] = round(batch / t, 2)
    if seeding_ab:
        for flag in ("1", "0"):
            os.environ["ZKE_NATIVE_REGEX"] = flag                          # read when a context opens
            cw = z.Context(c, None, device=0, max_batch=batch)
            cw.witness(packed, batch, want_witness=False)
            cw.profile(True)
            ms = []
            for _ in range(repeats):
                cw.witness(packed, batch, want_witness=False)
                ms.append(cw.profile_get()["witness"]["ms"])
            row["witness_ms_batch%d_native_regex_%s" % (batch, flag)] = round(statistics.median(ms[i] - (ms[i - 1] if i else 0) for i in range(len(ms))), 2)
            del cw
        os.environ.pop("ZKE_NATIVE_REGEX", None)
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
        raise SystemExit("app_bench needs a CUDA device")
    sizes = {"maxHeadersLength": a.headers, "maxBodyLength": a.body}
    rows = []
    for style in (1, 0):
        rows.append(bench("TwitterVerifier style %d" % style, dict(TWITTER_SPEC, regexStyle=style, **sizes), a.batch, a.repeats, twitter=True))
        rows.append(bench("app style %d" % style, dict(app_spec(style), **sizes), a.batch, a.repeats, seeding_ab=True))
        print(json.dumps(rows[-2:]), flush=True)
    res = dict(_gpu_info(), headers=a.headers, body=a.body, batch=a.batch, repeats=a.repeats, results=rows)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
