"""Device pairing arithmetic of the GPU batch verifier (zk-email-verify_b200/csrc/pairing.cuh) checked on the CPU under
ZKE_FF_EMULATE: the Fq12 tower operations against oracle/bn254.py, the sparse line product against the dense one, the
pairing (Miller loop + final exponentiation) against the library's host-only zke_pairing_alphabeta, bilinearity, the
fixture's vk_alphabeta_12, replayed line tables against the on-the-fly loop, and the G2 subgroup check."""
import ctypes, json, os, random, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import bn254

import zkemail_b200  # noqa: F401  (loads the library for zke_pairing_alphabeta)
from zkemail_b200 import _lib as L

Q, R = bn254.P, bn254.R
RM = 1 << 256
GOLD = os.path.join(ROOT, "tests", "golden", "proof_of_twitter")


def _build():
    out = os.path.join(tempfile.gettempdir(), "libzke_pairing_emulation_%d.so" % os.getuid())
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zk-email-verify_b200", "csrc"),
                           "-Wno-unknown-pragmas", os.path.join(ROOT, "tests", "pairing_emulation.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    arr = lambda x: (ctypes.c_uint32 * 8)(*[(x >> (32 * i)) & 0xffffffff for i in range(8)])
    inv = lambda m: ctypes.c_uint32((-pow(m, -1, 1 << 32)) % (1 << 32))
    lib.pe_set_consts(arr(Q), arr(RM % Q), arr(RM * RM % Q), inv(Q), arr(R), arr(RM % R), arr(RM * RM % R), inv(R))
    return lib


lib = _build()
mont = lambda x: (x % Q * RM % Q).to_bytes(32, "little")
unmont = lambda b: int.from_bytes(b, "little") * pow(RM, -1, Q) % Q


# tower coefficient (i, j) multiplies w^(2j + i); u = w^6 - 9 in the oracle's dense Fq[w]/(w^12 - 18 w^6 + 82)
def to_tower(f):
    out = b""
    for i in range(2):
        for j in range(3):
            n = 2 * j + i
            out += mont(f.c[n] + 9 * f.c[n + 6]) + mont(f.c[n + 6])
    return out


def from_tower(b):
    c = [0] * 12
    for i in range(2):
        for j in range(3):
            n, k = 2 * j + i, 64 * (3 * i + j)
            a0, a1 = unmont(b[k:k + 32]), unmont(b[k + 32:k + 64])
            c[n], c[n + 6] = a0 - 9 * a1, a1
    return bn254.F12(c)


def f12_op(which, a, b=None):
    out = ctypes.create_string_buffer(384)
    bb = to_tower(b) if isinstance(b, bn254.F12) else (b or bytes(384))
    lib.pe_f12(which, to_tower(a), bb, out)
    return from_tower(out.raw)


def g1b(p):
    return bytes(64) if p is None else mont(p[0]) + mont(p[1])


def g2b(p):
    return bytes(128) if p is None else mont(p[0][0]) + mont(p[0][1]) + mont(p[1][0]) + mont(p[1][1])


def pairing(p, q, final=True):
    out = ctypes.create_string_buffer(384)
    lib.pe_pairing(g1b(p), g2b(q), 1 if final else 0, out)
    return from_tower(out.raw)


def host_pairing(p, q):
    le = lambda v: v.to_bytes(32, "little")
    out = ctypes.create_string_buffer(384)
    assert L.zke_pairing_alphabeta(le(p[0]) + le(p[1]), le(q[0][0]) + le(q[0][1]) + le(q[1][0]) + le(q[1][1]), out) == 0
    # output: tower coefficients in standard form
    c = [0] * 12
    for i in range(2):
        for j in range(3):
            n, k = 2 * j + i, 64 * (3 * i + j)
            a0, a1 = int.from_bytes(out.raw[k:k + 32], "little"), int.from_bytes(out.raw[k + 32:k + 64], "little")
            c[n], c[n + 6] = a0 - 9 * a1, a1
    return bn254.F12(c)


def rand_f12(rng):
    return bn254.F12([rng.randrange(Q) for _ in range(12)])


def rand_pair(rng):
    return bn254.g1_mul(bn254.G1_GEN, rng.randrange(1, R)), bn254.g2_mul(bn254.G2_GEN, rng.randrange(1, R))


def test_tower_arithmetic_matches_oracle():
    rng = random.Random(11)
    for _ in range(4):
        a, b = rand_f12(rng), rand_f12(rng)
        assert f12_op(0, a, b) == a * b
        assert f12_op(1, a) == a * a
        assert f12_op(3, a) == a.inv()
        assert f12_op(4, a) == a ** Q
        assert f12_op(5, a) == a ** (Q * Q)
        assert f12_op(6, a) == a ** (Q ** 3)
    a = rand_f12(rng)
    assert f12_op(9, a) == a ** (Q ** 6)        # conjugation is the p^6-th power


def test_cyclotomic_square_on_cyclotomic_elements():
    rng = random.Random(12)
    for _ in range(3):
        a = rand_f12(rng)
        m = f12_op(9, a) * a.inv()                # a^(p^6 - 1)
        m = (m ** (Q * Q)) * m                    # ^(p^2 + 1): in the cyclotomic subgroup
        assert f12_op(2, m) == m * m
    x = rand_f12(rng)
    assert f12_op(2, x) != x * x                  # the formula is only valid on the subgroup


def test_sparse_line_product_equals_dense_product():
    rng = random.Random(13)
    for _ in range(4):
        a = rand_f12(rng)
        l = [(rng.randrange(Q), rng.randrange(Q)) for _ in range(3)]
        line_bytes = b"".join(mont(x) + mont(y) for x, y in l)
        # dense element: l0 at (0, 0), l1 at (1, 0) = w, l2 at (1, 1) = v w
        dense = bytearray(384)
        dense[0:64] = line_bytes[0:64]
        dense[192:256] = line_bytes[64:128]
        dense[256:320] = line_bytes[128:192]
        assert f12_op(7, a, line_bytes) == a * from_tower(bytes(dense))


def test_pairing_matches_host_pairing_on_random_pairs():
    rng = random.Random(14)
    for _ in range(8):
        p, q = rand_pair(rng)
        assert pairing(p, q) == host_pairing(p, q)


def test_pairing_is_bilinear():
    rng = random.Random(15)
    p, q = rand_pair(rng)
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    lhs = pairing(bn254.g1_mul(p, a), bn254.g2_mul(q, b))
    assert lhs == pairing(p, q) ** (a * b % R)
    assert lhs != pairing(p, q)
    # infinity on either side gives 1
    assert pairing(None, q) == bn254.F12.one() and pairing(p, None) == bn254.F12.one()


def test_pairing_reproduces_fixture_alphabeta():
    vkey = json.load(open(os.path.join(GOLD, "vkey.json")))
    alpha = bn254.g1_from_json(vkey["vk_alpha_1"])
    beta = bn254.g2_from_json(vkey["vk_beta_2"])
    e = pairing(alpha, beta)
    got = [[[None, None] for _ in range(3)] for _ in range(2)]
    for i in range(2):
        for j in range(3):
            n = 2 * j + i
            got[i][j] = [str((e.c[n] + 9 * e.c[n + 6]) % Q), str(e.c[n + 6])]
    assert got == vkey["vk_alphabeta_12"]


def test_replayed_lines_equal_on_the_fly_loop():
    rng = random.Random(16)
    (p1, q), (p2, _), (p3, q2) = rand_pair(rng), rand_pair(rng), rand_pair(rng)
    fly, both, only = (ctypes.create_string_buffer(384) for _ in range(3))
    lib.pe_replay(g1b(p1), g2b(q), g1b(p2), g2b(q2), g1b(p3), fly, both, only)
    assert from_tower(fly.raw) == pairing(p1, q, final=False)
    assert from_tower(only.raw) == pairing(p2, q, final=False)
    assert from_tower(both.raw) == pairing(p2, q, final=False) * pairing(p3, q2, final=False)


def _twist_point_outside_subgroup():
    for x0 in range(1, 60):
        x = (x0, 0)
        rhs = bn254.f2_add(bn254.f2_mul(bn254.f2_sqr(x), x), bn254.B2)
        a, b = rhs
        n = (a * a + b * b) % Q
        s = pow(n, (Q + 1) // 4, Q)
        if s * s % Q != n:
            continue
        for sgn in (s, Q - s):
            t = (a + sgn) * pow(2, -1, Q) % Q
            y0 = pow(t, (Q + 1) // 4, Q)
            if y0 * y0 % Q != t or y0 == 0:
                continue
            y = (y0, b * pow(2 * y0, -1, Q) % Q)
            if bn254.f2_sqr(y) == rhs:
                return (x, y)
    raise AssertionError("no twist point found")


def test_subgroup_check_agrees_with_oracle():
    rng = random.Random(17)
    for _ in range(3):
        q = bn254.g2_mul(bn254.G2_GEN, rng.randrange(1, R))
        assert lib.pe_g2_check(g2b(q)) == 3
    rogue = _twist_point_outside_subgroup()
    assert bn254.g2_is_on_curve(rogue) and bn254.g2_mul(rogue, R - 1) != bn254.g2_neg(rogue)
    assert lib.pe_g2_check(g2b(rogue)) == 1
    # a multiple of it is still outside (the cofactor does not divide the scalar)
    rogue3 = bn254.g2_add(bn254.g2_add(rogue, rogue), rogue)
    assert lib.pe_g2_check(g2b(rogue3)) == 1
    off = (rogue[0], bn254.f2_add(rogue[1], (1, 0)))
    assert lib.pe_g2_check(g2b(off)) == 0
    assert lib.pe_g2_check(g2b(None)) == 3
