"""Prepared phase-2 `.ptau` images written in Python on oracle/bn254.py - the independent restatement of the layout the
native reader (setup.cu) and the native toy writer (zke_ptau_toy) follow.

Sections: 1 header {n8q, q, power, ceremonyPower}; 2 tauG1 (2^(power+1) - 1 points); 3 tauG2, 4 alphaTauG1, 5 betaTauG1
(2^power each); 6 betaG2; 7 contributions (u32 count 0); 12-15 lTauG1, lTauG2, lAlphaTauG1, lBetaTauG1: the Lagrange bases
of the domains 1, 2, ..., 2^power back to back.  Points affine, Montgomery little-endian, G2 as x.c0, x.c1, y.c0, y.c1."""
from __future__ import annotations
import struct

from oracle import bn254

Q, R = bn254.P, bn254.R
MONT = pow(2, 256, Q)
G1 = (1, 2)
G2 = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
       11559732032986387107991004021392285783925812861821192530917403151452391805634),
      (8495653923123431417604973247489272438418190587263600148770280649306958101930,
       4082367875863433681332203403145435568316851327593401208105741076214120093531))
ORDER = (1, 2, 3, 4, 5, 6, 7, 12, 13, 14, 15)


def _fq(x: int) -> bytes:
    return (x * MONT % Q).to_bytes(32, "little")


def g1_bytes(p) -> bytes:
    return bytes(64) if p is None else _fq(p[0]) + _fq(p[1])


def g2_bytes(p) -> bytes:
    return bytes(128) if p is None else _fq(p[0][0]) + _fq(p[0][1]) + _fq(p[1][0]) + _fq(p[1][1])


def root_of_unity(log_n: int) -> int:
    """Primitive 2^log_n-th root of unity mod r (5 generates the multiplicative group)."""
    return pow(5, (R - 1) >> log_n, R)


def lagrange(tau: int, log_n: int) -> list[int]:
    """L_i(tau) = (tau^n - 1) / n * omega^i / (tau - omega^i) for the domain of size n = 2^log_n."""
    n = 1 << log_n
    w = root_of_unity(log_n)
    num = (pow(tau, n, R) - 1) * pow(n, -1, R) % R
    out, wi = [], 1
    for _ in range(n):
        out.append(num * wi * pow(tau - wi, -1, R) % R)
        wi = wi * w % R
    return out


def section_counts(power: int) -> dict:
    n = 1 << power
    return {2: (2 * n - 1, 64), 3: (n, 128), 4: (n, 64), 5: (n, 64), 6: (1, 128),
            12: (2 * n - 1, 64), 13: (2 * n - 1, 128), 14: (2 * n - 1, 64), 15: (2 * n - 1, 64)}


def write_ptau(power: int, tau: int | None = None, alpha: int = 0, beta: int = 0, overrides: dict | None = None):
    """Returns (file bytes, {section: (payload offset, payload size)}).  With tau = None the point sections are filled with
    the generators (a structurally valid file whose points are not a ceremony's: enough for the host reader).  `overrides`
    replaces section payloads (or header fields via key "header") to build malformed files."""
    overrides = overrides or {}
    cnt = section_counts(power)
    pay = {}
    pay[1] = overrides.get("header", struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<II", power, power))
    if tau is None:
        for s, (k, size) in cnt.items():
            pay[s] = (g1_bytes(G1) if size == 64 else g2_bytes(G2)) * k
    else:
        n = 1 << power
        pw = [pow(tau, i, R) for i in range(2 * n - 1)]
        lag = [v for k in range(power + 1) for v in lagrange(tau, k)]
        g1 = lambda ks: b"".join(g1_bytes(bn254.g1_mul(G1, k % R)) for k in ks)   # noqa: E731
        g2 = lambda ks: b"".join(g2_bytes(bn254.g2_mul(G2, k % R)) for k in ks)   # noqa: E731
        pay[2], pay[3] = g1(pw), g2(pw[:n])
        pay[4], pay[5], pay[6] = g1(alpha * v for v in pw[:n]), g1(beta * v for v in pw[:n]), g2([beta])
        pay[12], pay[13] = g1(lag), g2(lag)
        pay[14], pay[15] = g1(alpha * v for v in lag), g1(beta * v for v in lag)
    pay[7] = struct.pack("<I", 0)
    pay.update({k: v for k, v in overrides.items() if isinstance(k, int)})   # a value of None drops the section
    present = [s for s in ORDER if pay.get(s) is not None]
    out = bytearray(b"ptau" + struct.pack("<II", 1, len(present)))
    where = {}
    for s in present:
        out += struct.pack("<IQ", s, len(pay[s]))
        where[s] = (len(out), len(pay[s]))
        out += pay[s]
    return bytes(out), where
