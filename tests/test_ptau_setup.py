"""Host side of the Powers-of-Tau key setup (no GPU): the native `.ptau` reader against the Python writer of
tests/ptau_writer.py, its refusals, and the algebra behind the H points."""
import random
import struct

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from ptau_writer import Q, R, lagrange, root_of_unity, section_counts, write_ptau


@pytest.mark.parametrize("power", [1, 4, 11])
def test_reader_agrees_with_python_writer_on_every_section(power):
    data, where = write_ptau(power)
    info = z.ptau_info(data)
    assert info["power"] == power
    assert info["sections"] == {1: where[1], **{s: where[s] for s in where if s != 1}}
    for s, (k, size) in section_counts(power).items():
        assert where[s][1] == k * size
    # a writable buffer and a path are read the same way
    assert z.ptau_info(bytearray(data)) == info


def test_reader_maps_a_path(tmp_path):
    data, _ = write_ptau(3)
    p = tmp_path / "t.ptau"
    p.write_bytes(data)
    assert z.ptau_info(str(p)) == z.ptau_info(data)


def test_malformed_files_are_refused():
    good, where = write_ptau(4)
    with pytest.raises(L.ZkeError, match="bad magic"):
        z.ptau_info(b"zkey" + good[4:])
    bad_q = struct.pack("<I", 32) + (Q + 2).to_bytes(32, "little") + struct.pack("<II", 4, 4)
    with pytest.raises(L.ZkeError, match="not over the BN254 base field"):
        z.ptau_info(write_ptau(4, overrides={"header": bad_q})[0])
    with pytest.raises(L.ZkeError, match=r"truncated .ptau \(section 15\)"):
        z.ptau_info(good[:-10])
    with pytest.raises(L.ZkeError, match=r"section 3 \(tauG2\) has 1920 bytes, expected 2048 for power 4"):
        z.ptau_info(write_ptau(4, overrides={3: bytes(128 * 15)})[0])
    with pytest.raises(L.ZkeError, match=r"section 13 \(lTauG2\) is missing"):
        z.ptau_info(write_ptau(4, overrides={13: None})[0])
    big_power = struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<II", 5, 5)
    with pytest.raises(L.ZkeError, match=r"section 2 \(tauG1\) has .* expected .* for power 5"):
        z.ptau_info(write_ptau(4, overrides={"header": big_power})[0])
    with pytest.raises(L.ZkeError, match="appears twice"):
        off = where[7][0] - 12
        sec7 = good[off:off + 16]
        z.ptau_info(good[:8] + struct.pack("<I", struct.unpack("<I", good[8:12])[0] + 1) + good[12:] + sec7)


def test_file_too_small_for_the_circuit():
    c = z.Circuit("PackRegexReveal", [64, 21])      # domain 2^11: H needs the basis of size 2^12
    assert c.info.domain_log2 == 11
    with pytest.raises(L.ZkeError, match=r"power 11 is too small for this circuit: its domain 2\^11 needs power 12 or more"):
        z.ptau_info(write_ptau(11)[0], c)
    assert z.ptau_info(write_ptau(12)[0], c)["power"] == 12


def test_h_points_are_the_odd_entries_of_the_double_size_basis():
    """H_i = -L_i(tau/g) Z(tau) / 2 (the engine's quotient basis at delta = 1, setup_host.cpp) equals point 2i + 1 of the
    Lagrange basis of size 2N, with g a primitive 2N-th root of unity."""
    rng = random.Random(5)
    for log_n in (1, 3, 6):
        n = 1 << log_n
        g = root_of_unity(log_n + 1)
        omega = root_of_unity(log_n)
        assert g * g % R == omega
        for _ in range(3):
            tau = rng.randrange(2, R)
            big = lagrange(tau, log_n + 1)
            small_at = lagrange(tau * pow(g, -1, R) % R, log_n)
            z_tau = (pow(tau, n, R) - 1) % R
            for i in range(n):
                assert big[2 * i + 1] == (-small_at[i] * z_tau * pow(2, -1, R)) % R


def test_lagrange_basis_interpolates():
    """The Python basis (the layout's definition) sums to 1 and reproduces x at tau: sum L_i(tau) omega^i = tau."""
    tau = 123456789
    for log_n in (0, 2, 5):
        lag = lagrange(tau, log_n)
        w = root_of_unity(log_n)
        assert sum(lag) % R == 1
        assert sum(v * pow(w, i, R) for i, v in enumerate(lag)) % R == tau % R if log_n else True
