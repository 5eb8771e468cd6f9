"""Edge cases of the witness kernel's cooperative ops against the CPU oracle, bit for bit (run with `-m gpu`).

  * FpMul hint: every case of tests/test_bigdiv_hint.py's table of a shape in one batch, one email per case, so that each
    email's CTA decides its own mode and caches its own reciprocal: Barrett with 0, 1 and 2 corrections at t = 4, 32 and
    64 words and both normalisation shifts, P = b^(t-1), every fallback reason, Knuth's qhat decrements and add-backs,
    R = 0, R = P - 1, A = 0, limbs at or above 2^n, quotients beyond k limbs and a zero modulus.  Cluster widths 1 and 8
    (the cooperative ops run on rank 0), and the sequential hint alone (ZKE_COOP_FPMUL=0).
  * RSAVerifier65537(121, 17): 17 chained hints on one modulus (the reciprocal cache hits 16 times) for a 1024-bit, a
    2048-bit and a 2040-bit key (normalisation shift 8).
  * Regex seeding across the 896-position chunk boundaries of the 64-state and the compact mode (witness.cu: regex_coop):
    matches straddling positions 896 and 1792 with states >= 32 carried over, bytes >= 0x80 at the boundary, and a non-byte
    value just past it (tests/test_app_circuit.py: long_regex_messages, checked on the CPU there).

Every element's witness equals the oracle's, failing elements included, and its status is the oracle's first violated
constraint (-1 when all hold)."""
import ctypes
import functools
import hashlib

import pytest

import zkemail_b200 as z
from zkutil import oracle_witness, ref, ref_view
from test_app_circuit import LONG_LEN, LONG_REGEX, long_regex_messages
from test_bigdiv_hint import SHAPES, cases_of, expected, fpmul_circuit, must_fail

pytestmark = pytest.mark.gpu


def _oracle(c, inputs):
    """(the oracle's witness, its first violated constraint or -1)."""
    w = oracle_witness(c, inputs, check=False)
    return w.raw(), ref.zkref_check_r1cs(ctypes.byref(ref_view(c)), w.buf)


def _run(c, inputs, refs, names):
    """One batch on the GPU; every element against the oracle."""
    packed = b"".join(c.pack_inputs(x) for x in inputs)
    ctx = z.Context(c, None, device=0, max_batch=len(inputs))
    wt, status = ctx.witness(packed, len(inputs), raise_on_fail=False)
    ctx.close()
    m = 32 * c.info.n_vars
    bad = [f"{e} {names[e]}: status {status[e]} (oracle {first}), witness {'equal' if wt[m * e:m * (e + 1)] == w else 'differs'}"
           for e, (w, first) in enumerate(refs) if status[e] != first or wt[m * e:m * (e + 1)] != w]
    assert not bad, "elements differ from the oracle:\n" + "\n".join(bad)
    return wt


# ------------------------------------------------------------------------------------------------ FpMul hint
@functools.lru_cache(maxsize=None)
def _fpmul_batch(n, k):
    c = fpmul_circuit(n, k)
    rows = cases_of(n, k)
    inputs = [{"a": a, "b": b, "p": p} for _, _, a, b, p, _ in rows]
    refs = [_oracle(c, x) for x in inputs]
    assert [first >= 0 for _, first in refs] == [must_fail(*row[:5]) for row in rows]
    return c, rows, inputs, refs


@pytest.mark.parametrize("width,coop", [("1", "1"), ("8", "1"), ("1", "0"), ("8", "0")],
                         ids=["width1", "width8", "sequential-width1", "sequential-width8"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{n},{k}" for n, k in SHAPES])
def test_fpmul_hint_table(shape, width, coop, monkeypatch):
    monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    monkeypatch.setenv("ZKE_COOP_FPMUL", coop)
    c, rows, inputs, refs = _fpmul_batch(*shape)
    wt = _run(c, inputs, refs, [f"{row[5]}" for row in rows])
    first, count, _ = c.groups["out"]
    m = 32 * c.info.n_vars
    for e, (n, k, a, b, p, label) in enumerate(rows):
        got = [int.from_bytes(wt[m * e + 32 * (first + i):m * e + 32 * (first + i + 1)], "little") for i in range(count)]
        assert got == expected(n, k, a, b, p)[1], f"{e} {label}: out is not the remainder"


# ------------------------------------------------------------------------------------------------ RSA: chained hints
@functools.lru_cache(maxsize=None)
def _rsa_batch():
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding
    from test_templates_sha_rsa import MESSAGE, PUB_1024, SIG_1024
    c = z.Circuit("RSAVerifier65537", [121, 17])
    inputs = [{"signature": z.to_circom_bigint_bytes(SIG_1024), "modulus": z.to_circom_bigint_bytes(PUB_1024), "message": MESSAGE}]
    names = ["1024-bit fixture"]
    for bits in (2048, 2040):
        key = z.synthetic.generate_key(bits, seed=bits)
        data = b"chained FpMul hints, %d-bit key" % bits
        sig = int.from_bytes(key.sign(data, padding.PKCS1v15(), hashes.SHA256()), "big")
        modulus = key.public_key().public_numbers().n
        assert modulus.bit_length() == bits
        inputs.append({"signature": z.to_circom_bigint_bytes(sig), "modulus": z.to_circom_bigint_bytes(modulus),
                       "message": z.to_circom_bigint_bytes(int.from_bytes(hashlib.sha256(data).digest(), "big"))})
        names.append(f"{bits}-bit key")
    refs = [_oracle(c, x) for x in inputs]
    assert [first for _, first in refs] == [-1] * len(inputs)
    return c, inputs, refs, names


@pytest.mark.parametrize("width", ["1", "8"])
def test_rsa_chained_hints(width, monkeypatch):
    monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    monkeypatch.delenv("ZKE_COOP_FPMUL", raising=False)
    c, inputs, refs, names = _rsa_batch()
    _run(c, inputs, refs, names)


# ------------------------------------------------------------------------------------------------ regex chunk boundaries
@functools.lru_cache(maxsize=None)
def _regex_batch(style):
    c = z.Circuit.from_regex(LONG_REGEX, LONG_LEN)       # built under ZKE_REGEX_STYLE = style
    msgs = long_regex_messages()
    inputs = [{"msg": m} for m in msgs]
    refs = [_oracle(c, x) for x in inputs]
    # the non-byte value: the zk-regex shape does not range-check its message, the compact shape rejects it
    assert [first >= 0 for _, first in refs] == [False] * (len(msgs) - 1) + [style == "1"]
    return c, inputs, refs


@pytest.mark.parametrize("width", ["1", "8"])
@pytest.mark.parametrize("style", ["0", "1"], ids=["zkregex", "compact"])
def test_regex_seeding_across_chunk_boundaries(style, width, monkeypatch):
    monkeypatch.setenv("ZKE_REGEX_STYLE", style)
    monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    c, inputs, refs = _regex_batch(style)
    names = [f"message {e}" for e in range(len(inputs) - 1)] + ["non-byte value at position 897"]
    _run(c, inputs, refs, names)
