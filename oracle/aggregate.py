"""Aggregation of n Groth16 proofs under one key into one O(log n) proof (SnarkPack: TIPP + MIPP with KZG-committed keys).

TEST INFRASTRUCTURE (oracle) - never imported by the product path.  A plain-integer restatement, on bn254.py, of the
protocol written down in DESIGN.md ("Proof aggregation"): byte layout, transcript and checks.  The native prover
(aggregate.cu) and host verifier (aggregate_host.cpp) are compared against it.

Pairing values (GT) are those of snarkjs' vk_alphabeta_12: the reduced pairing raised to K = 2 z (6 z^2 + 3 z + 1).
"""
from __future__ import annotations

import hashlib

from . import bn254 as b

P, R = b.P, b.R
K_SNARKJS = 0x3bec47df15e307c81ea96b02d9d9e38d2e5d4e223ddedaf4
DOMAIN_TAG = b"zkemail-snarkpack-groth16-v1"
GT_BYTES, G1_BYTES, G2_BYTES = 384, 64, 128
ROUND_GT = ("ZL", "ZR", "TL", "TR", "UL", "UR", "TCL", "TCR", "UCL", "UCR")
HEAD_BYTES = 5 * GT_BYTES + G1_BYTES                      # T_AB U_AB T_C U_C Z_AB Z_C
ROUND_BYTES = len(ROUND_GT) * GT_BYTES + 2 * G1_BYTES    # ... ZCL ZCR
TAIL_BYTES = 4 * G1_BYTES + 3 * G2_BYTES + 2 * G2_BYTES + 2 * G1_BYTES   # A B C v1 v2 w1 w2, pi_v1 pi_v2 pi_w1 pi_w2


def agg_bytes(n: int) -> int:
    return HEAD_BYTES + (n.bit_length() - 1) * ROUND_BYTES + TAIL_BYTES


class AggError(ValueError):
    pass


# ---- encodings (standard form, little-endian; infinity = all zero, as zke_prove) ---------------------------------------
def fq_b(x: int) -> bytes:
    return x.to_bytes(32, "little")


def g1_b(pt) -> bytes:
    return bytes(64) if pt is None else fq_b(pt[0]) + fq_b(pt[1])


def g2_b(pt) -> bytes:
    return bytes(128) if pt is None else fq_b(pt[0][0]) + fq_b(pt[0][1]) + fq_b(pt[1][0]) + fq_b(pt[1][1])


def gt_b(f: b.F12) -> bytes:
    """Dense F12 -> the tower layout of vk_alphabeta_12: coefficient (i, j) = (c[n] + 9 c[n+6]) + c[n+6] u, n = 2j + i."""
    out = b""
    for i in range(2):
        for j in range(3):
            n = 2 * j + i
            out += fq_b((f.c[n] + 9 * f.c[n + 6]) % P) + fq_b(f.c[n + 6])
    return out


def _words(buf: bytes, count: int):
    ws = [int.from_bytes(buf[32 * k:32 * k + 32], "little") for k in range(count)]
    if any(w >= P for w in ws):
        raise AggError("coordinate not reduced")
    return ws


def gt_from(buf: bytes) -> b.F12:
    w = _words(buf, 12)
    c = [0] * 12
    for i in range(2):
        for j in range(3):
            n, k = 2 * j + i, 2 * (3 * i + j)
            c[n], c[n + 6] = w[k] - 9 * w[k + 1], w[k + 1]
    return b.F12(c)


def g1_from(buf: bytes):
    x, y = _words(buf, 2)
    pt = None if x == 0 and y == 0 else (x, y)
    if not b.g1_is_on_curve(pt):
        raise AggError("G1 point not on the curve")
    return pt


def g2_from(buf: bytes):
    w = _words(buf, 4)
    pt = None if not any(w) else ((w[0], w[1]), (w[2], w[3]))
    if not b.g2_is_on_curve(pt):
        raise AggError("G2 point not on the twist curve")
    if pt is not None and _g2_mul_raw(pt, R) is not None:   # bn254.g2_mul reduces its scalar mod r
        raise AggError("G2 point not in the order-r subgroup")
    return pt


def _g2_mul_raw(pt, k: int):
    res, add = None, pt
    while k:
        if k & 1:
            res = b.g2_add(res, add)
        add = b.g2_add(add, add)
        k >>= 1
    return res


def gt(f: b.F12) -> b.F12:
    return b.final_exponentiate(f) ** K_SNARKJS


def pair_prod(pairs) -> b.F12:
    """prod e(P, Q) over (G1, G2) pairs, one final exponentiation."""
    f = b.F12.one()
    for p1, q2 in pairs:
        f = f * b.miller_loop(q2, p1)
    return gt(f)


def g1_sum(pts):
    acc = None
    for p in pts:
        acc = b.g1_add(acc, p)
    return acc


def challenge(*parts: bytes) -> int:
    c = int.from_bytes(hashlib.sha256(b"".join(parts)).digest(), "little") % R
    if c == 0:
        raise AggError("zero challenge")
    return c


def vkey_bytes(vkey: dict) -> bytes:
    out = g1_b(b.g1_from_json(vkey["vk_alpha_1"]))
    for k in ("vk_beta_2", "vk_gamma_2", "vk_delta_2"):
        out += g2_b(b.g2_from_json(vkey[k]))
    return out + b"".join(g1_b(b.g1_from_json(p)) for p in vkey["IC"])


def publics_bytes(publics) -> bytes:
    return b"".join(fq_b(int(s)) for row in publics for s in row)


# ---- SRS ----------------------------------------------------------------------------------------------------------------
class Srs:
    """Powers of two independent secrets a, b: g^(a^i), g^(b^i) for i < 2 n_max and h^(a^i), h^(b^i) for i < n_max."""

    def __init__(self, a: int, bb: int, n_max: int):
        self.n_max = n_max
        self.g_a = [b.g1_mul(b.G1_GEN, pow(a, i, R)) for i in range(2 * n_max)]
        self.g_b = [b.g1_mul(b.G1_GEN, pow(bb, i, R)) for i in range(2 * n_max)]
        self.h_a = [b.g2_mul(b.G2_GEN, pow(a, i, R)) for i in range(n_max)]
        self.h_b = [b.g2_mul(b.G2_GEN, pow(bb, i, R)) for i in range(n_max)]

    def vk(self) -> dict:
        return {"protocol": "snarkpack", "curve": "bn128", "g": b.g1_to_json(self.g_a[0]), "h": b.g2_to_json(self.h_a[0]),
                "g_a": b.g1_to_json(self.g_a[1]), "g_b": b.g1_to_json(self.g_b[1]),
                "h_a": b.g2_to_json(self.h_a[1]), "h_b": b.g2_to_json(self.h_b[1])}


def _check_n(n: int, n_max: int | None = None):
    if n < 2 or n > 8192 or n & (n - 1):
        raise AggError(f"the number of proofs must be a power of two from 2 to 8192, not {n}")
    if n_max is not None and n > n_max:
        raise AggError(f"{n} proofs exceed the SRS size {n_max}")


def _fold_polys(xs, r_inv, n):
    """Coefficients of f_v(X) = prod_j (1 + x_j^-1 (X / r)^(n / 2^(j+1))) and d_i, F_w(X) = X^n sum_i d_i X^i with
    sum_i d_i X^i = prod_j (1 + x_j X^(n / 2^(j+1))): key i is folded with the product of the challenges of the rounds that
    took it from the right half."""
    cv, dw = [1] * n, [1] * n
    for i in range(n):
        for j, x in enumerate(xs):
            if (i >> (len(xs) - 1 - j)) & 1:
                cv[i] = cv[i] * pow(x, -1, R) % R
                dw[i] = dw[i] * x % R
        cv[i] = cv[i] * pow(r_inv, i, R) % R
    return cv, [0] * n + dw


def _quotient(coeffs, z):
    """(f(X) - f(z)) / (X - z) by synthetic division; coefficients low to high."""
    q = [0] * (len(coeffs) - 1)
    acc = 0
    for i in range(len(coeffs) - 1, 0, -1):
        acc = (acc * z + coeffs[i]) % R
        q[i - 1] = acc
    return q


def _poly_eval(coeffs, z):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * z + c) % R
    return acc


def aggregate(srs: Srs, vkey: dict, proofs, publics) -> bytes:
    """proofs: [(A, B, C)] affine points (bn254 tuples); publics: [[int]] per proof -> the aggregate's bytes."""
    n = len(proofs)
    _check_n(n, srs.n_max)
    if len(publics) != n:
        raise AggError("one public-signal vector per proof")
    n_pub = len(vkey["IC"]) - 1
    if any(len(s) != n_pub for s in publics):
        raise AggError(f"every proof needs {n_pub} public signals")
    A = [p[0] for p in proofs]
    B = [p[1] for p in proofs]
    C = [p[2] for p in proofs]
    v1, v2, w1, w2 = srs.h_a[:n], srs.h_b[:n], srs.g_a[n:2 * n], srs.g_b[n:2 * n]
    t_ab = pair_prod(list(zip(A, v1)) + list(zip(w1, B)))
    u_ab = pair_prod(list(zip(A, v2)) + list(zip(w2, B)))
    t_c = pair_prod(zip(C, v1))
    u_c = pair_prod(zip(C, v2))
    com = gt_b(t_ab) + gt_b(u_ab) + gt_b(t_c) + gt_b(u_c)
    r = challenge(DOMAIN_TAG, vkey_bytes(vkey), n.to_bytes(4, "little"), com, publics_bytes(publics))
    r_inv = pow(r, -1, R)
    A = [b.g1_mul(a, pow(r, i, R)) for i, a in enumerate(A)]
    C = [b.g1_mul(c, pow(r, i, R)) for i, c in enumerate(C)]
    v1 = [b.g2_mul(v, pow(r_inv, i, R)) for i, v in enumerate(v1)]
    v2 = [b.g2_mul(v, pow(r_inv, i, R)) for i, v in enumerate(v2)]
    out = com + gt_b(pair_prod(zip(A, B))) + g1_b(g1_sum(C))
    x, beta, xs = r, 1, []
    while len(A) > 1:
        h = len(A) // 2
        AL, AR, BL, BR, CL, CR = A[:h], A[h:], B[:h], B[h:], C[:h], C[h:]
        v1L, v1R, v2L, v2R, w1L, w1R, w2L, w2R = v1[:h], v1[h:], v2[:h], v2[h:], w1[:h], w1[h:], w2[:h], w2[h:]
        msg = b"".join(gt_b(pair_prod(pp)) for pp in (
            zip(AR, BL), zip(AL, BR),
            list(zip(AR, v1L)) + list(zip(w1R, BL)), list(zip(AL, v1R)) + list(zip(w1L, BR)),
            list(zip(AR, v2L)) + list(zip(w2R, BL)), list(zip(AL, v2R)) + list(zip(w2L, BR)),
            zip(CR, v1L), zip(CL, v1R), zip(CR, v2L), zip(CL, v2R)))
        msg += g1_b(b.g1_mul(g1_sum(CR), beta)) + g1_b(b.g1_mul(g1_sum(CL), beta))
        x = challenge(fq_b(x), msg)
        xi = pow(x, -1, R)
        xs.append(x)
        out += msg
        A = [b.g1_add(l, b.g1_mul(rr, x)) for l, rr in zip(AL, AR)]
        C = [b.g1_add(l, b.g1_mul(rr, x)) for l, rr in zip(CL, CR)]
        B = [b.g2_add(l, b.g2_mul(rr, xi)) for l, rr in zip(BL, BR)]
        v1 = [b.g2_add(l, b.g2_mul(rr, xi)) for l, rr in zip(v1L, v1R)]
        v2 = [b.g2_add(l, b.g2_mul(rr, xi)) for l, rr in zip(v2L, v2R)]
        w1 = [b.g1_add(l, b.g1_mul(rr, x)) for l, rr in zip(w1L, w1R)]
        w2 = [b.g1_add(l, b.g1_mul(rr, x)) for l, rr in zip(w2L, w2R)]
        beta = beta * (1 + xi) % R
    final = g1_b(A[0]) + g2_b(B[0]) + g1_b(C[0]) + g2_b(v1[0]) + g2_b(v2[0]) + g1_b(w1[0]) + g1_b(w2[0])
    z = challenge(fq_b(x), final)
    cv, cw = _fold_polys(xs, r_inv, n)
    qv, qw = _quotient(cv, z), _quotient(cw, z)
    msm1 = lambda pts, sc: g1_sum(b.g1_mul(p, s) for p, s in zip(pts, sc))   # noqa: E731
    msm2 = lambda pts, sc: _g2_sum(b.g2_mul(p, s) for p, s in zip(pts, sc))  # noqa: E731
    out += final + g2_b(msm2(srs.h_a, qv)) + g2_b(msm2(srs.h_b, qv)) + g1_b(msm1(srs.g_a, qw)) + g1_b(msm1(srs.g_b, qw))
    assert len(out) == agg_bytes(n)
    return out


def _g2_sum(pts):
    acc = None
    for p in pts:
        acc = b.g2_add(acc, p)
    return acc


def _g2_from_json_checked(v):
    pt = b.g2_from_json(v)
    return g2_from(g2_b(pt))


def verify(agg_vk: dict, vkey: dict, publics, agg: bytes) -> bool:
    """True iff `agg` proves that n valid Groth16 proofs under `vkey` exist for these public signals (n = len(publics))."""
    try:
        return _verify(agg_vk, vkey, publics, agg)
    except (AggError, KeyError, ValueError, AssertionError, IndexError, TypeError):
        return False


def _verify(agg_vk, vkey, publics, agg):
    n = len(publics)
    _check_n(n)
    if len(agg) != agg_bytes(n):
        return False
    n_pub = len(vkey["IC"]) - 1
    pubs = [[int(s) for s in row] for row in publics]
    if any(len(row) != n_pub or any(not 0 <= s < R for s in row) for row in pubs):
        return False
    g = g1_from(g1_b(b.g1_from_json(agg_vk["g"])))
    h = _g2_from_json_checked(agg_vk["h"])
    g_a, g_b = (g1_from(g1_b(b.g1_from_json(agg_vk[k]))) for k in ("g_a", "g_b"))
    h_a, h_b = (_g2_from_json_checked(agg_vk[k]) for k in ("h_a", "h_b"))
    alpha = g1_from(g1_b(b.g1_from_json(vkey["vk_alpha_1"])))
    beta2, gamma2, delta2 = (_g2_from_json_checked(vkey[k]) for k in ("vk_beta_2", "vk_gamma_2", "vk_delta_2"))
    ic = [g1_from(g1_b(b.g1_from_json(p))) for p in vkey["IC"]]

    off = 0

    def take(nbytes):
        nonlocal off
        off += nbytes
        return agg[off - nbytes:off]

    com = take(4 * GT_BYTES)
    t_ab, u_ab, t_c, u_c = (gt_from(com[GT_BYTES * k:GT_BYTES * (k + 1)]) for k in range(4))
    z_ab0 = z_ab = gt_from(take(GT_BYTES))
    z_c0 = z_c = g1_from(take(G1_BYTES))
    r = challenge(DOMAIN_TAG, vkey_bytes(vkey), n.to_bytes(4, "little"), com, publics_bytes(pubs))
    x, beta, xs = r, 1, []
    for _ in range(n.bit_length() - 1):
        msg = take(ROUND_BYTES)
        m = {name: gt_from(msg[GT_BYTES * k:GT_BYTES * (k + 1)]) for k, name in enumerate(ROUND_GT)}
        zcl = g1_from(msg[len(ROUND_GT) * GT_BYTES:][:G1_BYTES])
        zcr = g1_from(msg[len(ROUND_GT) * GT_BYTES + G1_BYTES:])
        x = challenge(fq_b(x), msg)
        xi = pow(x, -1, R)
        xs.append(x)
        z_ab = z_ab * m["ZL"] ** x * m["ZR"] ** xi
        t_ab = t_ab * m["TL"] ** x * m["TR"] ** xi
        u_ab = u_ab * m["UL"] ** x * m["UR"] ** xi
        t_c = t_c * m["TCL"] ** x * m["TCR"] ** xi
        u_c = u_c * m["UCL"] ** x * m["UCR"] ** xi
        z_c = b.g1_add(z_c, b.g1_add(b.g1_mul(zcl, x), b.g1_mul(zcr, xi)))
        beta = beta * (1 + xi) % R
    final = take(TAIL_BYTES - 2 * G2_BYTES - 2 * G1_BYTES)
    fa, fc, fw1, fw2 = (g1_from(final[o:o + G1_BYTES]) for o in (0, 192, 512, 576))
    fb, fv1, fv2 = (g2_from(final[o:o + G2_BYTES]) for o in (64, 256, 384))
    pv1, pv2 = g2_from(take(G2_BYTES)), g2_from(take(G2_BYTES))
    pw1, pw2 = g1_from(take(G1_BYTES)), g1_from(take(G1_BYTES))
    z = challenge(fq_b(x), final)

    # GIPA final relations
    if z_ab != pair_prod([(fa, fb)]):
        return False
    if t_ab != pair_prod([(fa, fv1), (fw1, fb)]) or u_ab != pair_prod([(fa, fv2), (fw2, fb)]):
        return False
    if z_c != b.g1_mul(fc, beta) or t_c != pair_prod([(fc, fv1)]) or u_c != pair_prod([(fc, fv2)]):
        return False
    # KZG openings of the folded keys at z: v = h^f_v(tau), w = g^F_w(tau) for tau = a, b
    cv, cw = _fold_polys(xs, pow(r, -1, R), n)
    fvz, fwz = _poly_eval(cv, z), _poly_eval(cw, z)
    one = b.F12.one()
    for tau_g, key, pi in ((g_a, fv1, pv1), (g_b, fv2, pv2)):
        if pair_prod([(b.g1_add(tau_g, b.g1_neg(b.g1_mul(g, z))), pi), (b.g1_neg(g), b.g2_add(key, b.g2_neg(b.g2_mul(h, fvz))))]) != one:
            return False
    for tau_h, key, pi in ((h_a, fw1, pw1), (h_b, fw2, pw2)):
        if pair_prod([(pi, b.g2_add(tau_h, b.g2_neg(b.g2_mul(h, z)))), (b.g1_neg(b.g1_add(key, b.g1_neg(b.g1_mul(g, fwz)))), h)]) != one:
            return False
    # Groth16 in aggregated form: Z_AB = e(alpha, beta)^(sum r^i) e(sum_i r^i vk_x_i, gamma) e(Z_C, delta)
    rp = [pow(r, i, R) for i in range(n)]
    coeff = [sum(rp) % R] + [sum(rp[i] * pubs[i][j] for i in range(n)) % R for j in range(n_pub)]
    vk_x = g1_sum(b.g1_mul(p, c) for p, c in zip(ic, coeff))
    return z_ab0 == pair_prod([(b.g1_mul(alpha, coeff[0]), beta2), (vk_x, gamma2), (z_c0, delta2)])
