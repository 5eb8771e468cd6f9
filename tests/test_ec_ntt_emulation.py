"""Point transform and per-point scaling of zk-email-verify_b200/csrc/ec_ntt.cuh (the kernels behind ptau_prepare and
ptau_contribute) checked on the CPU under ZKE_FF_EMULATE against oracle/bn254.py, in G1 and G2.

Input points are multiples [t_j] G of known scalars (t_j = 0 is the point at infinity), so the oracle's transform is a
transform of the scalars followed by one multiplication per output point."""
import ctypes, os, random, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import bn254

Q, R = bn254.P, bn254.R
RM = 1 << 256
G1 = (1, 2)


def _build():
    out = os.path.join(tempfile.gettempdir(), "libzke_ec_ntt_emulation_%d.so" % os.getuid())
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zk-email-verify_b200", "csrc"),
                           "-Wno-unknown-pragmas", os.path.join(ROOT, "tests", "ec_ntt_emulation.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    arr = lambda x: (ctypes.c_uint32 * 8)(*[(x >> (32 * i)) & 0xffffffff for i in range(8)])
    lib.en_set_consts(arr(Q), arr(RM % Q), arr(RM * RM % Q), ctypes.c_uint32((-pow(Q, -1, 1 << 32)) % (1 << 32)))
    return lib


lib = _build()
mont = lambda x: (x % Q * RM % Q).to_bytes(32, "little")
unmont = lambda b: int.from_bytes(b, "little") * pow(RM, -1, Q) % Q


def enc(pt, g2):
    if pt is None:
        return bytes(128 if g2 else 64)
    if g2:
        return mont(pt[0][0]) + mont(pt[0][1]) + mont(pt[1][0]) + mont(pt[1][1])
    return mont(pt[0]) + mont(pt[1])


def dec(b, g2):
    if not any(b):
        return None
    v = [unmont(b[32 * i:32 * i + 32]) for i in range(len(b) // 32)]
    return ((v[0], v[1]), (v[2], v[3])) if g2 else (v[0], v[1])


def mul(k, g2):
    k %= R
    if k == 0:
        return None
    return bn254.g2_mul(bn254.G2_GEN, k) if g2 else bn254.g1_mul(G1, k)


def words(ks):
    return b"".join(int(k).to_bytes(32, "little") for k in ks)


def root_of_unity(log_n):
    return pow(5, (R - 1) >> log_n, R)


def transform(t, g2):
    n = len(t)
    log_n = n.bit_length() - 1
    w_inv = pow(root_of_unity(log_n), -1, R)
    tw = words(pow(w_inv, j, R) for j in range(max(1, n // 2)))
    size = 128 if g2 else 64
    out = ctypes.create_string_buffer(size * n)
    lib.en_transform(int(g2), log_n, b"".join(enc(mul(x, g2), g2) for x in t), tw, words([pow(n, -1, R)]), out)
    return [dec(out.raw[size * i:size * (i + 1)], g2) for i in range(n)]


def oracle_transform(t):
    n = len(t)
    w_inv = pow(root_of_unity(n.bit_length() - 1), -1, R)
    n_inv = pow(n, -1, R)
    return [n_inv * sum(pow(w_inv, i * j, R) * x for j, x in enumerate(t)) % R for i in range(n)]


def test_point_transform_matches_the_oracle():
    rng = random.Random(29)
    for g2 in (False, True):
        for log_n in range(7):
            n = 1 << log_n
            t = [rng.randrange(R) for _ in range(n)]
            for j in rng.sample(range(n), min(n, 2)):
                t[j] = 0                                    # infinity among the inputs
            assert transform(t, g2) == [mul(x, g2) for x in oracle_transform(t)], (g2, n)
        # a constant input transforms to one point and n - 1 infinities; all-infinity stays all-infinity
        assert transform([7] * 8, g2) == [mul(7, g2)] + [None] * 7
        assert transform([0] * 4, g2) == [None] * 4


def test_per_point_scaling_matches_the_oracle():
    rng = random.Random(31)
    ks = [0, 1, 2, 3, R - 1, R - 2, R, (1 << 254) - 1, (1 << 253) + 1, (1 << 200) - 1, int("01" * 126, 2), int("10" * 126, 2),
          int("0111" * 62, 2), ((1 << 100) - 1) << 120] + [rng.randrange(R) for _ in range(10)]
    for g2 in (False, True):
        base = [rng.randrange(1, R) for _ in ks]
        base[3] = 0                                         # infinity times anything is infinity
        size = 128 if g2 else 64
        out = ctypes.create_string_buffer(size * len(ks))
        lib.en_scale(int(g2), len(ks), b"".join(enc(mul(b, g2), g2) for b in base), words(ks), out)
        got = [dec(out.raw[size * i:size * (i + 1)], g2) for i in range(len(ks))]
        assert got == [mul(b * k, g2) for b, k in zip(base, ks)], g2
