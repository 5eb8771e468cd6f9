"""The FpMul big-integer hint, (q, r) = divmod(A * B, P) on n-bit limbs, against exact Python integers on a table of edge
cases (the GPU witness kernel runs the same table in tests/test_gpu_witness_edges.py).

The hint has two code paths: Knuth's algorithm D on 32-bit words (csrc/bigdiv.hpp: bd_knuth_div, fpmul_hint_words),
shared by the host export zke_selftest_fpmul_hint and the witness kernel's sequential path; and the kernel's cooperative
Barrett reduction (csrc/witness.cu: fpmul_coop, Handbook of Applied Cryptography 14.42), which falls back to the sequential
path when Barrett's preconditions fail.  The models below mirror both on 32-bit words and report which branch each case
takes: qhat decrements and add-backs of the division, the Barrett mode, the reason for a fallback, the reciprocal mu and the
number of corrective subtractions.  Random operands never reach most of these branches (an add-back has probability about
2 / 2^32 per quotient digit, a second Barrett correction needs a modulus just above b^(t-1)), so the table constructs them.

The ground truth is always divmod on Python integers; the expected limbs are its quotient and remainder re-split into n-bit
limbs and truncated to k limbs, which is what the hint writes (bd_extract) and what the oracle writes (big_extract)."""
import ctypes
import functools
import random

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkutil import oracle_witness, ref, ref_view

BW = 32
BASE = 1 << BW
MASK = BASE - 1
MAXW = 80                      # bigdiv.hpp: BIGDIV_MAXW
SHAPES = [(32, 5), (121, 9), (121, 17)]


def words(x, count):
    return [(x >> (BW * i)) & MASK for i in range(count)]


def value(ws):
    return sum(v << (BW * i) for i, v in enumerate(ws))


def n_words(x):
    return (x.bit_length() + BW - 1) // BW


def split(x, n, k):
    """x as k limbs of n bits, truncated (bd_extract / big_extract)."""
    return [(x >> (n * i)) & ((1 << n) - 1) for i in range(k)]


def join(limbs, n):
    """The integer the circuit's limbs stand for: limbs may be at or above 2^n."""
    return sum(v << (n * i) for i, v in enumerate(limbs))


def width(n, k):
    """W of fpmul_hint_words / fpmul_coop: words per operand."""
    return (n * k + 256 + 31) // 32


# ------------------------------------------------------------------------------------------------ models
def knuth_div(U, UL, P, t, stats):
    """Mirror of bd_knuth_div: U[0..UL] (UL + 2 words) divided by P[0..t) (top word non-zero), both lists modified in place
    as the C code does.  Returns Q[0..UL]; U[0..t) holds the remainder.  Counts qhat decrements and add-backs in `stats`."""
    Q = [0] * (UL + 1)
    s = 0
    while ((P[t - 1] << s) & 0x80000000) == 0:
        s += 1
    stats["s"] = s
    if s:
        for i in range(t - 1, 0, -1):
            P[i] = ((P[i] << s) | (P[i - 1] >> (BW - s))) & MASK
        P[0] = (P[0] << s) & MASK
        for i in range(UL, 0, -1):
            U[i] = ((U[i] << s) | (U[i - 1] >> (BW - s))) & MASK
        U[0] = (U[0] << s) & MASK
    if t == 1:
        rem = 0
        for j in range(UL, -1, -1):
            cur = (rem << BW) | U[j]
            Q[j] = (cur // P[0]) & MASK
            rem = cur % P[0]
            U[j] = 0
        U[0] = rem
    else:
        v1, v2 = P[t - 1], P[t - 2]
        for j in range(UL - t, -1, -1):
            num = (U[j + t] << BW) | U[j + t - 1]
            qhat, rhat = divmod(num, v1)
            while qhat >= BASE or qhat * v2 > ((rhat << BW) | U[j + t - 2]):
                qhat -= 1
                stats["decrements"] += 1
                rhat += v1
                if rhat >= BASE:
                    break
            borrow = carry = 0
            for i in range(t):
                prod = qhat * P[i] + carry
                carry = prod >> BW
                sub = (U[i + j] - (prod & MASK) - borrow) & (2**64 - 1)
                U[i + j] = sub & MASK
                borrow = (sub >> BW) & 1
            sub = (U[j + t] - carry - borrow) & (2**64 - 1)
            U[j + t] = sub & MASK
            if (sub >> BW) & 1:
                qhat -= 1
                stats["addbacks"] += 1
                c = 0
                for i in range(t):
                    sm = U[i + j] + P[i] + c
                    U[i + j] = sm & MASK
                    c = sm >> BW
                U[j + t] = (U[j + t] + c) & MASK
            Q[j] = qhat & MASK
    if s:
        for i in range(t):
            U[i] = (U[i] >> s) | (((U[i + 1] << (BW - s)) & MASK) if i + 1 <= UL else 0)
    return Q


def _operands(n, k, a, b, p):
    """A, B, P as fpmul_hint_words assembles them (bd_add_shifted: each limb's 256 bits, the sum mod b^W)."""
    W = width(n, k)
    mod = 1 << (BW * W)
    return W, join(a, n) % mod, join(b, n) % mod, join(p, n) % mod


def _new_stats():
    return {"decrements": 0, "addbacks": 0, "s": None}


def hint_words(n, k, a, b, p):
    """Mirror of fpmul_hint_words (the sequential path): (q, r, stats); q and r are the integers the limbs are cut from."""
    W, A, B, P = _operands(n, k, a, b, p)
    assert W <= MAXW and 0 < n <= 128
    stats = _new_stats()
    UL = 2 * W
    U = words(A * B, UL) + [0, 0]
    t = n_words(P)
    if t == 0:                 # division by zero: zeros, the constraints reject
        return 0, 0, stats
    Q = knuth_div(U, UL, words(P, t), t, stats)
    return value(Q), value(U[:t]), stats


def reciprocal(P, t, stats):
    """mu as fpmul_coop computes it: bd_knuth_div of b^(2t) by P, the low t + 1 quotient words kept."""
    U = [0] * (2 * t) + [1, 0]
    Q = knuth_div(U, 2 * t, words(P, t), t, stats)
    assert len(Q) == 2 * t + 1 and all(v == 0 for v in Q[t + 1:])     # the division writes no word above t
    return value(Q[:t + 1])


def fpmul_coop(n, k, a, b, p, rounds=3):
    """Mirror of fpmul_coop's mode decision and Barrett step.  Returns a dict: mode ("barrett" / "sequential"), reason for
    a fallback, t, s, mu, corrections, the Knuth statistics of the division that ran (mu's or the sequential one), q, r."""
    W, A, B, P = _operands(n, k, a, b, p)
    t = n_words(P)
    out = {"t": t, "mu": None, "corrections": None, "reason": None}
    if t == 0:
        out["reason"] = "P=0"
    elif t < 4:
        out["reason"] = "t<=3"
    elif A >= BASE**t:
        out["reason"] = "A>=b^t"
    elif B >= BASE**t:
        out["reason"] = "B>=b^t"
    elif P == BASE**(t - 1):
        out["reason"] = "P=b^(t-1)"
    if out["reason"]:
        q, r, stats = hint_words(n, k, a, b, p)
        out.update(mode="sequential", q=q, r=r, knuth=stats, s=stats["s"])
        return out
    stats = _new_stats()
    mu = reciprocal(P, t, stats)
    X = A * B
    q3 = ((X >> (BW * (t - 1))) * mu) >> (BW * (t + 1))
    top = BASE**(t + 1)
    R = (X - q3 * P) % top     # X - q3 P mod b^(t+1), the words fpmul_coop subtracts
    Q = q3
    corrections = 0
    for _ in range(rounds):
        if R < P:
            break
        R = (R - P) % top
        Q = (Q + 1) % top
        corrections += 1
    out.update(mode="barrett", q=Q, r=R, mu=mu, corrections=corrections, knuth=stats, s=stats["s"])
    return out


# ------------------------------------------------------------------------------------------------ case table
CLASSES = [
    *(f"barrett {c} corrections t={t}" for c in (0, 1, 2) for t in (4, 32, 64)),
    "barrett s=0", "barrett s>0", "reciprocal add-back",
    "P=b^(t-1) t=4", "P=b^(t-1) t=64",
    "fallback t<=3", "fallback P=0", "fallback A>=b^t", "fallback B>=b^t",
    "sequential qhat decrement", "sequential add-back",
    "R=0", "R=P-1", "A=0", "limb>=2^n", "quotient overflow",
]


def classes(n, k, a, b, p):
    """The classes the models put a case in."""
    m = fpmul_coop(n, k, a, b, p)
    _, A, B, P = _operands(n, k, a, b, p)
    t, out = m["t"], set()
    if m["mode"] == "barrett":
        out.add(f"barrett {m['corrections']} corrections t={t}")
        out.add("barrett s=0" if m["s"] == 0 else "barrett s>0")
        if m["knuth"]["addbacks"]:
            out.add("reciprocal add-back")
    else:
        r = m["reason"]
        out.add(f"P=b^(t-1) t={t}" if r == "P=b^(t-1)" else f"fallback {r}")
        if m["knuth"]["decrements"]:
            out.add("sequential qhat decrement")
        if m["knuth"]["addbacks"]:
            out.add("sequential add-back")
    if P and A * B % P == 0:
        out.add("R=0")
    if P and A * B % P == P - 1:
        out.add("R=P-1")
    if A == 0:
        out.add("A=0")
    if any(v >> n for v in (*a, *b, *p)):
        out.add("limb>=2^n")
    if P and A * B // P >> (n * k):
        out.add("quotient overflow")
    return out


def _search(rng, n, k, label, gen, tries=20000):
    for _ in range(tries):
        A, B, P = gen()
        case = (split(A, n, k), split(B, n, k), split(P, n, k))
        if label in classes(n, k, *case):
            return case
    raise AssertionError(f"no {label} case found")


@functools.lru_cache(maxsize=None)
def cases_of(n, k):
    """[(n, k, a_limbs, b_limbs, p_limbs, label)] for one shape, built deterministically."""
    rng = random.Random(n * 1000 + k)
    rows = []
    add = lambda label, a, b, p: rows.append((n, k, list(a), list(b), list(p), label))
    lim = lambda x: split(x, n, k)
    ts = [t for t in (4, 32, 64) if BW * t <= n * k]

    for t in ts:
        top0 = lambda: BASE**t - 1 - rng.getrandbits(BW * t - 1)                   # top bit set: s = 0
        topx = lambda: (rng.randrange(2, 1 << 31) << (BW * (t - 1))) + rng.getrandbits(BW * (t - 1))   # 1 <= s <= 30
        near = lambda: BASE**(t - 1) + 1 + rng.getrandbits(BW * (t - 2))          # just above b^(t-1): s = 31
        below = lambda P: rng.randrange(P)
        for corr in (0, 1):
            for mk in (top0, topx):
                def gen(mk=mk):
                    P = mk()
                    return below(P), below(P), P
                add(f"barrett {corr} corrections t={t}", *_search(rng, n, k, f"barrett {corr} corrections t={t}", gen))

        def gen2():
            P = near()
            return (BASE**t - 1 - rng.getrandbits(16 * t), BASE**t - 1 - rng.getrandbits(16 * t), P)
        add(f"barrett 2 corrections t={t}", *_search(rng, n, k, f"barrett 2 corrections t={t}", gen2))

        # the reciprocal division's first digit overestimates by one: P = 2^31 b^(t-1) + 1 (v2 = 0, the +1 below)
        P = (1 << 31) * BASE**(t - 1) + 1
        add("reciprocal add-back", lim(rng.randrange(P)), lim(rng.randrange(P)), lim(P))
        # R = 0, R = P - 1 and A = 0 at both shifts
        for P in (top0(), topx()):
            B = rng.randrange(1, P)
            add("R=0", lim(P), lim(B), lim(P))
            while True:
                B = rng.randrange(2, P)
                try:
                    add("R=P-1", lim(-pow(B, -1, P) % P), lim(B), lim(P))
                    break
                except ValueError:
                    continue
            add("A=0", lim(0), lim(B), lim(P))

    # P = b^(t-1) exactly: its reciprocal b^(t+1) does not fit t + 1 words
    for t in (4, 64):
        if BW * t <= n * k:
            P = BASE**(t - 1)
            bmax = min(BASE**t, 1 << (n * k - BW)) - 1                             # the quotient fits k limbs
            add(f"P=b^(t-1) t={t}", lim(BASE**t - 1 - rng.getrandbits(BW * t - 2)), lim(bmax), lim(P))
            add(f"P=b^(t-1) t={t}", lim(rng.randrange(P)), lim(rng.randrange(BASE**t)), lim(P))

    # sequential path: small moduli, operands above b^t, and Knuth's rare branches
    for t in (1, 2, 3):
        P = rng.getrandbits(BW * t) | (1 << (BW * t - 1 - rng.randrange(8)))
        add("fallback t<=3", lim(rng.randrange(P)), lim(rng.randrange(P)), lim(P))
    add("fallback P=0", lim(rng.getrandbits(n * k - 1)), lim(rng.getrandbits(n * k - 1)), lim(0))
    t = 4
    P = BASE**t - rng.getrandbits(BW * t - 1)
    add("fallback A>=b^t", lim(BASE**t + rng.getrandbits(n * k - 2 * BW - 2)), lim(rng.getrandbits(BW)), lim(P))
    add("fallback B>=b^t", lim(rng.randrange(1, BASE)), lim(BASE**t + rng.getrandbits(n * k - 2 * BW - 2)), lim(P))

    def gen_dec():
        tt = rng.randrange(2, 4)
        P = rng.getrandbits(BW * tt) | 1 << (BW * tt - 1 - rng.randrange(32))
        return rng.randrange(P), rng.randrange(P), P
    add("sequential qhat decrement", *_search(rng, n, k, "sequential qhat decrement", gen_dec))
    # add-back (Hacker's Delight, divmnu64's test vector scaled to t words): P = 2^31 b^(t-1) + 1 and a dividend at or
    # above b^t, with B = 1 (the public circuit does not range-check a, b or p, so A >= b^t is a legal input)
    P = (1 << 31) * BASE**(t - 1) + 1
    add("sequential add-back", lim(BASE**t), lim(1), lim(P))
    add("sequential add-back", lim(1), lim(0x7fffffff * BASE**t + 0x80000000 * BASE**(t - 1)), lim(P))

    # limbs at or above 2^n (a, b and p are not range-checked): the integers they stand for still fit the hint's words
    P = BASE**t - 1 - rng.getrandbits(BW * t - 1)
    a = lim(rng.randrange(P))
    b = lim(rng.randrange(P))
    a[0] = 1 << n
    b[1] += (1 << n) + 3
    add("limb>=2^n", a, b, lim(P))
    p = lim(P)
    p[0] = 1 << n
    add("limb>=2^n", lim(rng.randrange(P)), lim(rng.randrange(P)), p)

    # quotient beyond k limbs: the hint truncates, the constraints reject
    add("quotient overflow", lim((1 << n * k) - 1), lim((1 << n * k) - 1), lim(3))
    add("quotient overflow", lim(BASE**t + 12345), lim((1 << n * k) - 1 - rng.getrandbits(BW)), lim(BASE**t - 5))
    return rows


CASES = [c for shape in SHAPES for c in cases_of(*shape)]
CASE_IDS = [f"{n},{k}:{i}:{label}" for i, (n, k, _, _, _, label) in enumerate(CASES)]


def expected(n, k, a, b, p):
    """(q limbs, r limbs) from divmod on Python integers; zeros for P = 0."""
    A, B, P = join(a, n), join(b, n), join(p, n)
    q, r = divmod(A * B, P) if P else (0, 0)
    return split(q, n, k), split(r, n, k)


def must_fail(n, k, a, b, p):
    """The constraints reject a zero modulus and a quotient beyond k limbs (which the hint truncates)."""
    return bool(classes(n, k, a, b, p) & {"fallback P=0", "quotient overflow"})


def selftest(n, k, a, b, p):
    enc = lambda xs: b"".join(v.to_bytes(32, "little") for v in xs)
    q, r = ctypes.create_string_buffer(32 * k), ctypes.create_string_buffer(32 * k)
    assert L.zke_selftest_fpmul_hint(n, k, enc(a), enc(b), enc(p), q, r) == 0
    dec = lambda buf: [int.from_bytes(buf.raw[32 * i:32 * i + 32], "little") for i in range(k)]
    return dec(q), dec(r)


# ------------------------------------------------------------------------------------------------ tests
def test_table_is_complete():
    """Every case is in the class its label names, and every class has cases."""
    counts = {c: 0 for c in CLASSES}
    for n, k, a, b, p, label in CASES:
        got = classes(n, k, a, b, p)
        assert label in got, f"({n}, {k}) {label}: the models put it in {sorted(got)}"
        for c in got:
            counts[c] += 1
    print("\nFpMul hint cases per class (%d cases):" % len(CASES))
    for c in CLASSES:
        print(f"  {counts[c]:3d}  {c}")
    assert all(counts.values()), [c for c, v in counts.items() if not v]


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_models_equal_divmod(case):
    n, k, a, b, p, _ = case
    want_q, want_r = expected(n, k, a, b, p)
    m = fpmul_coop(n, k, a, b, p)
    assert (split(m["q"], n, k), split(m["r"], n, k)) == (want_q, want_r)
    q, r, _ = hint_words(n, k, a, b, p)
    assert (split(q, n, k), split(r, n, k)) == (want_q, want_r)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_host_hint_equals_divmod(case):
    """zke_selftest_fpmul_hint: fpmul_hint_words, the code the kernel's sequential path runs."""
    n, k, a, b, p, _ = case
    assert selftest(n, k, a, b, p) == expected(n, k, a, b, p)


@functools.lru_cache(maxsize=None)
def fpmul_circuit(n, k):
    return z.Circuit("FpMul", [n, k])


def oracle_run(n, k, a, b, p):
    """(oracle witness, first violated constraint or -1)."""
    c = fpmul_circuit(n, k)
    w = oracle_witness(c, {"a": a, "b": b, "p": p}, check=False)
    return w, ref.zkref_check_r1cs(ctypes.byref(ref_view(c)), w.buf)


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{n},{k}" for n, k in SHAPES])
def test_oracle_agrees_and_rejects(shape):
    """The oracle's own hint writes the same q and r; the constraints hold on every case except a zero modulus and a
    quotient beyond k limbs."""
    for n, k, a, b, p, label in cases_of(*shape):
        w, first = oracle_run(n, k, a, b, p)
        assert w.values("out") == expected(n, k, a, b, p)[1], label
        assert (first >= 0) == must_fail(n, k, a, b, p), f"{label}: first violated constraint {first}"


def test_power_of_b_modulus_takes_the_sequential_path():
    """P = b^(t-1): the division fpmul_coop would use for the reciprocal leaves b^(t+1) - 1 in its t + 1 quotient words
    (the true reciprocal b^(t+1) needs t + 2), so the kernel detects this modulus and runs the sequential division."""
    for t in (4, 9, 64):
        assert reciprocal(BASE**(t - 1), t, _new_stats()) == BASE**(t + 1) - 1
        n, k = 121, 17
        m = fpmul_coop(n, k, split(BASE**t - 1, n, k), split(BASE**t - 2, n, k), split(BASE**(t - 1), n, k))
        assert (m["mode"], m["reason"]) == ("sequential", "P=b^(t-1)")


def test_barrett_needs_its_second_correction():
    """One correction round is not enough on the 2-correction cases (the bound of HAC 14.42 is tight)."""
    for n, k, a, b, p, label in CASES:
        if label.startswith("barrett 2"):
            assert split(fpmul_coop(n, k, a, b, p, rounds=1)["r"], n, k) != expected(n, k, a, b, p)[1]
