"""Phase 1 of the Powers-of-Tau ceremony on the GPU (ptau_new, ptau_contribute, ptau_prepare, verify_ptau) against the
native toy writer (ptau_toy, known secrets), the independent Python writer (tests/ptau_writer.py), tampered files, and
end to end through Zkey.from_ptau to a proof equal to the CPU oracle's."""
import struct

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkutil import oracle_prove, oracle_setup
from ptau_writer import Q, R, g2_bytes, write_ptau
from oracle import bn254

pytestmark = pytest.mark.gpu

T1 = (0x1F2E3D4C5B6A79880123456789ABCDEF0FEDCBA98765432, 0x2468ACE013579BDF2468ACE013579BDF, 0x0DDBA11CAFEBABE5EED)
T2 = (0x7E57AB1E * 10 ** 50 + 11, 0xA1FA * 10 ** 40 + 3, 0xBE7A * 10 ** 44 + 9)
PROD = tuple(a * b % R for a, b in zip(T1, T2))
SIZE = {2: 64, 3: 128, 4: 64, 5: 64, 6: 128, 12: 64, 13: 128, 14: 64, 15: 64}


def _sections(data) -> dict:
    n = struct.unpack_from("<I", data, 8)[0]
    pos, out = 12, {}
    for _ in range(n):
        t, size = struct.unpack_from("<IQ", data, pos)
        out[t] = bytes(data[pos + 12:pos + 12 + size])
        pos += 12 + size
    return out


def _phase1(data) -> dict:
    return {s: v for s, v in _sections(data).items() if s < 12}


def _patched(data, sec, dst, src=None, point=None):
    """`data` with point `dst` of section `sec` replaced by point `src` of the same section, or by the bytes `point`"""
    out = bytearray(data)
    n = struct.unpack_from("<I", out, 8)[0]
    pos = 12
    for _ in range(n):
        t, size = struct.unpack_from("<IQ", out, pos)
        if t == sec:
            ps, off = SIZE[sec], pos + 12
            new = point if point is not None else bytes(out[off + ps * src:off + ps * (src + 1)])
            out[off + ps * dst:off + ps * (dst + 1)] = new
            return bytes(out)
        pos += 12 + size
    raise KeyError(sec)


def _swapped(data, sec, i, j):
    a = _sections(data)[sec]
    ps = SIZE[sec]
    return _patched(_patched(data, sec, i, point=a[ps * j:ps * (j + 1)]), sec, j, point=a[ps * i:ps * (i + 1)])


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


@pytest.mark.parametrize("power", [1, 4, 11, 16])
def test_contribute_and_prepare_equal_the_native_writer(power):
    new = z.ptau_new(power)
    c1, _ = z.ptau_contribute(new, T1)
    toy1 = z.ptau_toy(power, *T1)
    assert _sections(c1) == _phase1(toy1)
    c2, _ = z.ptau_contribute(c1, T2)
    toy2 = z.ptau_toy(power, *PROD)
    assert _sections(c2) == _phase1(toy2)
    assert z.ptau_prepare(c1) == toy1
    assert z.ptau_prepare(c2) == toy2


@pytest.mark.parametrize("power", [1, 4])
def test_prepare_equals_the_python_writer(power):
    c1, _ = z.ptau_contribute(z.ptau_new(power), T1)
    assert bytes(z.ptau_prepare(c1)) == write_ptau(power, *T1)[0]


def test_contributing_to_a_prepared_file():
    toy = z.ptau_toy(4, *T1)
    marked = bytearray(toy)
    c, _ = z.ptau_contribute(marked, T2)
    assert sorted(_sections(c)) == [1, 2, 3, 4, 5, 6, 7]
    assert _sections(c)[7] == _sections(toy)[7]
    assert _sections(c) == _phase1(z.ptau_toy(4, *PROD))
    for bad, what in ((0, "zero"), (1, "one"), (R, "not below the group order r")):
        with pytest.raises(L.ZkeError, match=f"secret alpha is {what}"):
            z.ptau_contribute(toy, (T2[0], bad, T2[2]))
    rnd, receipt = z.ptau_contribute(toy)
    assert z.verify_ptau(rnd) and z.verify_ptau(z.ptau_prepare(rnd))
    assert z.verify_ptau(rnd, prev=toy, receipt=receipt)


def test_verify_accepts_honest_files():
    new = z.ptau_new(4)
    c1, _ = z.ptau_contribute(new, T1)
    for f in (new, c1, z.ptau_prepare(c1), z.ptau_prepare(new), z.ptau_toy(5, *T2)):
        ok, why = z.ptau_report(f, rand=bytes(range(16)))
        assert ok and why == "", why


def test_verify_rejects_tampered_files():
    c1, _ = z.ptau_contribute(z.ptau_new(4), T1)
    prep = z.ptau_prepare(c1)
    rogue = g2_bytes(_twist_point_outside_subgroup())
    cases = {
        "tauG1 i <- i+1": (_patched(c1, 2, 5, 6), "(tauG1)"),
        "tauG2 i <- i+1": (_patched(c1, 3, 2, 3), "(tauG2)"),
        "alphaTauG1 i <- i+1": (_patched(c1, 4, 2, 3), "(alphaTauG1)"),
        "betaTauG1 i <- i+1": (_patched(c1, 5, 2, 3), "(betaTauG1)"),
        "betaG2 <- tauG2[1]": (_patched(c1, 6, 0, point=_sections(c1)[3][128:256]), "(betaG2)"),
        "tauG1[0]": (_patched(c1, 2, 0, 1), "point 0 is not the G1 generator"),
        "twist point": (_patched(c1, 3, 2, point=rogue), "(tauG2): point 2 is not in the order-r subgroup"),
    }
    for s in (12, 13, 14, 15):   # points 1 and 2 of the size-4 basis (it starts at point 3)
        cases[f"Lagrange {s}"] = (_swapped(prep, s, 4, 5), f"section {s} (")
    for name, (bad, reason) in cases.items():
        ok, why = z.ptau_report(bad, rand=bytes(range(16)))
        assert not ok, f"{name}: tampered file accepted"
        assert reason in why, f"{name}: {why}"


def test_link_to_the_previous_file():
    new = z.ptau_new(3)
    c1, r1 = z.ptau_contribute(new, T1)
    c2, r2 = z.ptau_contribute(c1, T2)
    assert z.verify_ptau(c1, prev=new, receipt=r1)
    assert z.verify_ptau(c2, prev=c1, receipt=r2)
    assert z.verify_ptau(z.ptau_prepare(c2), prev=c1, receipt=r2)
    cases = {
        "another contribution's receipt": (c2, c1, r1, "(tauG1): point 1 is not the previous file's"),
        "unrelated file": (z.ptau_toy(3, T2[0] + 1, *T2[1:]), c1, r2, "is not the previous file's"),
        "receipt at infinity": (c2, c1, bytes(128) + r2[128:], "[tau]_2 is infinity"),
        "receipt off the subgroup": (c2, c1, r2[:256] + g2_bytes(_twist_point_outside_subgroup()), "[beta]_2 is not in the order-r subgroup"),
        "different power": (c2, z.ptau_new(4), r2, "power"),
    }
    for name, (nxt, prev, receipt, reason) in cases.items():
        ok, why = z.ptau_report(nxt, prev=prev, receipt=receipt)
        assert not ok, f"{name}: accepted"
        assert reason in why, f"{name}: {why}"


def test_ceremony_to_proof():
    """new -> contribute -> contribute -> prepare -> verify -> Zkey.from_ptau -> contribute(delta) -> proof == oracle's."""
    c = z.Circuit("Sha256Bytes", [64])
    delta = 0xD17A * 10 ** 60 + 7
    c1, r1 = z.ptau_contribute(z.ptau_new(c.info.domain_log2 + 1), T1)
    c2, r2 = z.ptau_contribute(c1, T2)
    prep = z.ptau_prepare(c2)
    assert z.verify_ptau(prep) and z.verify_ptau(prep, prev=c1, receipt=r2)
    key = z.Zkey.from_ptau(c, prep).contribute(delta.to_bytes(32, "little"))
    padded, plen = z.sha256_pad(b"phase one", 64)
    inputs = {"paddedIn": list(padded), "paddedInLength": plen}
    ctx = z.Context(c, key, device=0, max_batch=1)
    wt, status = ctx.witness(c.pack_inputs(inputs), 1)
    assert status == [-1]
    r, s = 1234567, 7654321
    proofs, publics, _ = ctx.prove(1, r.to_bytes(32, "little") + s.to_bytes(32, "little"))
    ctx.close()
    assert proofs == oracle_prove(c, oracle_setup(c, PROD + (1, delta)), wt, r, s)
    proof, pubs = z.proof_to_json(proofs, publics, c.info.n_public)
    vk = key.vkey()
    assert z.verify(vk, pubs, proof)
    assert z.Verifier(vk).verify_batch([pubs], [proof]) == [True]
