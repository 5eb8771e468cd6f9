"""The GPU prover and witness kernel against the CPU oracle, bit for bit, in every configuration the engine switches to
by batch or domain size (run with `-m gpu`).  Everything goes through the C ABI; the references are the oracle's witness,
constraint check and prover (tests/zkutil.py) and the pairing check of oracle/bn254.py.

  * Prover regimes: generated R1CS instances (tests/r1cs_gen.py) at every domain from 2^10 to 2^20 except 2^15, each
    with its own NTT pass split and H multi-exponentiation window, on adversarial witness scalars and points; two template
    circuits inside the c = 17 window with witnesses from the GPU kernel.
  * Proving lanes: 10 emails on 8 lanes (two lanes take two emails), 7 on 3 lanes, the single-stream lane form, and the
    pipelined submit / collect path.
  * Witness cluster widths 1, 2, 4 and 8 (CTAs per email), forced and chosen by batch size, with and without the lowering's
    native SHA-256 op, regex state seeding and cooperative FpMul; tampered batch elements name the oracle's first
    violated constraint.
"""
import ctypes
import functools
import random

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from oracle import bn254
from r1cs_gen import generate
from zkutil import oracle_prove, oracle_witness, product_sections, ref, ref_view

pytestmark = pytest.mark.gpu

R = z.FR_MODULUS
R_S = (0x2B1D0E5F6A7C8D9E0F1A2B3C4D5E6F708192A3B4C5D6E7F8, 0x7F6E5D4C3B2A19080F1E2D3C4B5A69788796A5B4C3D2E1F0)


def _rs(n, base=0):
    return b"".join((R_S[0] + base + e).to_bytes(32, "little") + (R_S[1] + 3 * (base + e)).to_bytes(32, "little")
                    for e in range(n))


def _assert_proof(c, zk, proof, publics, witness, k=0):
    """proof == the oracle's proof of `witness` at the k-th (r, s) of _rs, and the pairing check accepts it."""
    r, s = R_S[0] + k, R_S[1] + 3 * k
    assert proof == oracle_prove(c, product_sections(zk), witness, r, s, threads=16), "GPU proof differs from the oracle's"
    pj, pubs = z.proof_to_json(proof, publics, c.info.n_public)
    assert bn254.groth16_verify(zk.vkey(), pubs, pj)


# ------------------------------------------------------------------------------------------------ prover regimes
# domain -> NTT passes (ntt.cu: plan; the first passes strided, the last not) and H window c (msm.cu: msm_config_full,
# precomputed table).  The two-level digit sort of the H buckets (msm_sort.cuh) starts at c = 17.
REGIMES = [
    (10, "5+5, c = 12"),
    (11, "6+5, c = 12"),
    (12, "6+6, c = 12"),
    (13, "7+6, c = 12"),
    (14, "7+7, c = 12"),
    (16, "8+8, c = 17"),
    (17, "6+6+5, c = 17"),
    (18, "6+6+6, c = 17"),
    (19, "7+6+6, c = 17"),
    (20, "7+7+6, c = 20"),
]


@pytest.mark.parametrize("log_n", [r[0] for r in REGIMES], ids=[f"2^{k}: {d}" for k, d in REGIMES])
def test_generated_circuit_proof_equals_the_oracle(log_n):
    """More than 32 768 identical points under one small scalar (both extra reduction passes of a witness bucket), equal
    and opposite points in one bucket, points at infinity, scalars 0, 1, r - 1, (r -+ 1) / 2 and all-ones windows."""
    g = generate(log_n, seed=log_n)
    c = z.Circuit.from_r1cs(g["blob"])
    assert c.info.domain_log2 == log_n
    zk = z.Zkey(c, seed=100 + log_n)
    ctx = z.Context(c, zk, device=0, max_batch=1)
    ctx.load_witness(g["witness"], 1)
    proof, publics, status = ctx.prove(1, _rs(1, log_n))
    ctx.close()
    assert status == [-1]
    _assert_proof(c, zk, proof, publics, g["witness"], log_n)


def _sha_inputs(n, msgs):
    out = []
    for m in msgs:
        padded, plen = z.sha256_pad(m, n)
        out.append({"paddedIn": list(padded), "paddedInLength": plen})
    return out


def _rsa_input():
    from test_templates_sha_rsa import MESSAGE, PUB_1024, SIG_1024
    return {"signature": z.to_circom_bigint_bytes(SIG_1024), "modulus": z.to_circom_bigint_bytes(PUB_1024), "message": MESSAGE}


@pytest.mark.parametrize("template,params,log_n", [("Sha256Bytes", [128], 16), ("RSAVerifier65537", [121, 17], 18)],
                         ids=["Sha256Bytes(128) 2^16: 8+8, c = 17", "RSAVerifier65537(121, 17) 2^18: 6+6+6, c = 17"])
def test_template_circuit_in_the_c17_window(template, params, log_n):
    c = z.Circuit(template, params)
    assert c.info.domain_log2 == log_n
    inputs = _sha_inputs(128, [b"regimes at c = 17"])[0] if template == "Sha256Bytes" else _rsa_input()
    zk = z.Zkey(c, seed=200 + log_n)
    ctx = z.Context(c, zk, device=0, max_batch=1)
    wt, status = ctx.witness(c.pack_inputs(inputs), 1)
    assert status == [-1] and wt == oracle_witness(c, inputs).raw()
    proof, publics, _ = ctx.prove(1, _rs(1, 7))
    ctx.close()
    _assert_proof(c, zk, proof, publics, wt, 7)


# ------------------------------------------------------------------------------------------------ proving lanes
N_LANE_EMAILS = 10


@pytest.fixture(scope="module")
def lanes_setup():
    """Sha256Bytes(64) (2^15): 10 distinct messages, their GPU witnesses and the oracle's proofs at 10 distinct (r, s)."""
    c = z.Circuit("Sha256Bytes", [64])
    zk = z.Zkey(c, seed=64)
    inputs = _sha_inputs(64, [b"lane %d " % e * (e // 2 + 1) for e in range(N_LANE_EMAILS)])
    packed = b"".join(c.pack_inputs(i) for i in inputs)
    ctx = z.Context(c, None, device=0, max_batch=N_LANE_EMAILS)
    wt, status = ctx.witness(packed, N_LANE_EMAILS)
    ctx.close()
    m = c.info.n_vars
    assert status == [-1] * N_LANE_EMAILS and len({wt[32 * m * e:32 * m * (e + 1)] for e in range(N_LANE_EMAILS)}) == N_LANE_EMAILS
    sec = product_sections(zk)
    want = [oracle_prove(c, sec, wt[32 * m * e:32 * m * (e + 1)], R_S[0] + e, R_S[1] + 3 * e, threads=16)
            for e in range(N_LANE_EMAILS)]
    return c, zk, packed, wt, want


def _proofs(raw, n):
    return [raw[256 * e:256 * (e + 1)] for e in range(n)]


def test_lanes_and_stream_split(lanes_setup, monkeypatch):
    c, zk, packed, wt, want = lanes_setup
    n = N_LANE_EMAILS
    monkeypatch.delenv("ZKE_LANES", raising=False)
    monkeypatch.delenv("ZKE_SPLIT_STREAMS", raising=False)
    ctx = z.Context(c, zk, device=0, max_batch=n)
    assert L.zke_ctx_set_lanes(ctx.handle, 64) == 8          # eight lanes opened: emails 8 and 9 reuse lanes 0 and 1
    ctx.load_witness(wt, n)
    proofs, _, status = ctx.prove(n, _rs(n))
    assert status == [-1] * n and _proofs(proofs, n) == want, "8 lanes, two streams each"
    assert L.zke_ctx_set_lanes(ctx.handle, 3) == 3           # lanes 0, 1, 2 take three, two and two emails
    proofs, _, _ = ctx.prove(7, _rs(7))
    assert _proofs(proofs, 7) == want[:7], "3 lanes"
    assert L.zke_ctx_set_lanes(ctx.handle, 8) == 8
    monkeypatch.setenv("ZKE_SPLIT_STREAMS", "0")              # read by every prove call
    proofs, _, _ = ctx.prove(n, _rs(n))
    assert _proofs(proofs, n) == want, "8 lanes, one stream each"
    monkeypatch.setenv("ZKE_SPLIT_STREAMS", "1")
    ctx.submit(packed, n, _rs(n))
    proofs, publics, status = ctx.collect()
    assert status == [-1] * n and _proofs(proofs, n) == want, "submit / collect"
    npub = c.info.n_public
    m = c.info.n_vars
    assert publics == b"".join(wt[32 * m * e + 32:32 * m * e + 32 * (1 + npub)] for e in range(n))
    ctx.close()


# ------------------------------------------------------------------------------------------------ witness cluster widths
@functools.lru_cache(maxsize=None)
def _circuit_cases(name):
    """(circuit, distinct inputs, their oracle witnesses)."""
    rnd = random.Random(name)
    if name in ("sha128", "sha192"):
        n = int(name[3:])
        c = z.Circuit("Sha256Bytes", [n])
        inputs = _sha_inputs(n, [b"", b"cluster widths", bytes(range(n - 9)), b"\xff" * 64])
    elif name == "fpmul":
        c = z.Circuit("FpMul", [121, 17])
        inputs = []
        lim = lambda x: [(x >> (121 * i)) & ((1 << 121) - 1) for i in range(17)]
        for _ in range(3):
            p = rnd.getrandbits(2048) | (1 << 2047) | 1
            inputs.append({"a": lim(rnd.randrange(p)), "b": lim(rnd.randrange(p)), "p": lim(p)})
    elif name == "poseidon":
        c = z.Circuit("Poseidon", [2])
        inputs = [{"inputs": [1, 2]}, {"inputs": [0, R - 1]}, {"inputs": [rnd.randrange(R), rnd.randrange(R)]}]
    else:                               # email, email_compact
        params = [640, 768, 121, 17, 0, 0, 0, 0, 1] + ([1] if name == "email_compact" else [])
        c = z.Circuit("EmailVerifier", params)
        key = z.synthetic.generate_key(seed=3)
        inputs = []
        for i in range(3):
            dk = z.verify_dkim_signature(z.synthetic.make_signed_email(40 + i, key, body_len=512),
                                         resolver=lambda n_, t: [z.synthetic.key_record(key)])
            inputs.append(z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": 640, "maxBodyLength": 768}))
    return c, inputs, [oracle_witness(c, i).raw() for i in inputs]


@functools.lru_cache(maxsize=None)
def _tampered(name):
    """An EmailVerifier input that fails, and the first constraint the oracle's check finds violated in its witness."""
    c, inputs, _ = _circuit_cases(name)
    bad = dict(inputs[1])
    if name == "email":
        body = list(bad["emailBody"])
        body[7] = str((int(body[7]) + 1) % 128)
        bad["emailBody"] = body
    else:                               # a broken bh= tag
        hdr = list(bad["emailHeader"])
        hdr[int(bad["bodyHashIndex"]) - 2] = str(ord("-"))
        bad["emailHeader"] = hdr
    w = oracle_witness(c, bad, check=False)
    first = ref.zkref_check_r1cs(ctypes.byref(ref_view(c)), w.buf)
    assert first >= 0
    return bad, first


def _run_witness(c, inputs, refs, order, bad=None):
    """Witness of the batch `order` (indices into inputs; None = the tampered input) == the oracle, element by element."""
    packed = b"".join(c.pack_inputs(inputs[k] if k is not None else bad[0]) for k in order)
    ctx = z.Context(c, None, device=0, max_batch=len(order))
    wt, status = ctx.witness(packed, len(order), raise_on_fail=False)
    ctx.close()
    m = c.info.n_vars
    for e, k in enumerate(order):
        if k is None:
            assert status[e] == bad[1], f"element {e}: first violated constraint {status[e]}, the oracle's is {bad[1]}"
        else:
            assert status[e] == -1 and wt[32 * m * e:32 * m * (e + 1)] == refs[k], f"element {e} differs from the oracle"


WIDTHS = [1, 2, 4, 8]


@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("name", ["email", "email_compact", "sha192", "fpmul", "poseidon"])
def test_witness_at_forced_cluster_width(name, width, monkeypatch):
    """ZKE_WITNESS_CLUSTER, read when a context opens: each width is its own padded stream with its own barriers
    (tests/test_regimes_host.py checks the four streams differ); width 1 is a launch without clusters."""
    monkeypatch.setenv("ZKE_WITNESS_CLUSTER", str(width))
    c, inputs, refs = _circuit_cases(name)
    if name == "email":
        _run_witness(c, inputs, refs, [0, None, 2], _tampered(name))
    elif name == "email_compact":
        _run_witness(c, inputs, refs, [None, 0], _tampered(name))
    else:
        _run_witness(c, inputs, refs, list(range(len(inputs))))


@pytest.mark.parametrize("batch", [9, 33, 67], ids=["9: width 4", "33: width 2", "67: width 1 on 132 SMs"])
@pytest.mark.parametrize("name", ["sha128", "fpmul"])
def test_witness_at_default_cluster_width(name, batch, monkeypatch):
    """The width chosen by max_batch (engine.cu: upload_program): 8 up to 8 emails, 4 up to 32, 2 while two CTAs per
    email fit the SMs, else 1.  A handful of distinct inputs tiled over the whole batch."""
    monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    c, inputs, refs = _circuit_cases(name)
    _run_witness(c, inputs, refs, [e % len(inputs) for e in range(batch)])


@pytest.mark.parametrize("width", [1, 8])
@pytest.mark.parametrize("switch,name", [("ZKE_NATIVE_SHA", "sha192"), ("ZKE_NATIVE_REGEX", "email"), ("ZKE_COOP_FPMUL", "fpmul")],
                         ids=["native_sha_off", "regex_seeding_off", "coop_fpmul_off"])
def test_witness_without_a_lowering_substitution(switch, name, width, monkeypatch):
    monkeypatch.setenv("ZKE_WITNESS_CLUSTER", str(width))
    monkeypatch.setenv(switch, "0")
    c, inputs, refs = _circuit_cases(name)
    _run_witness(c, inputs, refs, list(range(len(inputs))))
