"""The oracle side of intra-proof sharding (DESIGN.md 6 (ii)), on the CPU: what each of G GPUs contributes to one proof.

A GPU of rank r in a world of G sums five multi-exponentiations over its share of the key and returns them as a 388-byte
partial (A, B1, C, H: 64 bytes each, B2: 128 bytes, then the first violated row of its rows, 0xffffffff for none):

  * A, B1, C and B2 over the point range [m r / G, m (r + 1) / G) of the m wires;
  * H over the column set {g M + r M / G + j : 0 <= g < G, 0 <= j < M / G}, M = N / G: the columns of every block of M
    positions that the engine's column layout gives the rank (not a contiguous range).

The CPU oracle's prover (oracle/zkref_groth16.c, zkref_groth16_prove) has no notion of a share, but its key can be masked:
with alpha1, beta1, delta1, beta2 and delta2 and every point outside the rank's share set to infinity, its assembly

    pi_A = alpha1 + A + r delta1        pi_B = beta2 + B2 + s delta2        pi_B1 = beta1 + B1 + s delta1
    pi_C = C + H + s pi_A + r pi_B1 - r s delta1

reduces to  (r, s) = (0, 0):                     pi_A = A, pi_B = B2, pi_C = C + H
            (0, 0), the whole C array masked:    pi_C = H
            (0, 0), the whole H array masked:    pi_C = C
            (1, 0), C and H masked:              pi_C = pi_B1 = B1

so three oracle proofs give a rank's five partial points.  The tests here pin that extraction and the layout against the
product's host combine (zke_shard_combine_raw): the G partials of G = 2, 4 and 8 add up to the oracle's unsharded proof,
and a flagged row in any one partial turns the result into that row's "Assert Failed".  tests/test_gpu_shard_one_device.py
compares the GPU ranks' partials with oracle_partials()."""
import ctypes

import numpy as np
import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from r1cs_gen import generate
from zkutil import oracle_prove, oracle_setup

NO_ROW = 0xFFFFFFFF
KEY_POINTS = ("alpha1", "beta1", "delta1", "beta2", "delta2")


def point_range(n_vars: int, rank: int, world: int) -> range:
    """The wires whose A, B1, C and B2 points rank `rank` sums (zke_shard_end: [m r / G, m (r + 1) / G))."""
    return range(n_vars * rank // world, n_vars * (rank + 1) // world)


def column_positions(n: int, rank: int, world: int) -> np.ndarray:
    """The positions of the H scalars rank `rank` computes: its M / G columns of every block of M = N / G positions."""
    if n % (world * world):
        raise ValueError("the column layout needs N to be a multiple of world^2")
    m, cols = n // world, n // (world * world)
    return (np.arange(world)[:, None] * m + rank * cols + np.arange(cols)[None, :]).reshape(-1)


def row_owner(row: int, n: int, world: int) -> int:
    """The rank whose column range holds constraint row `row` (the rank that checks it)."""
    m = n // world
    return (row % m) // (m // world)


def _mask(section: bytes, size: int, keep) -> bytes:
    """`section` (points of `size` bytes) with every point whose index is not in `keep` set to infinity (all zeros)."""
    pts = np.frombuffer(section, dtype=np.uint8).reshape(-1, size)
    out = np.zeros_like(pts)
    idx = np.asarray(keep, dtype=np.int64)
    out[idx] = pts[idx]
    return out.tobytes()


def mask_key(sec: dict, n_vars: int, log_n: int, rank: int, world: int, drop=()) -> dict:
    """A copy of the key sections `sec` (zkutil.oracle_setup / product_sections) reduced to rank `rank`'s share: the five
    fixed points at infinity, A / B1 / C / B2 outside the point range and H outside the column set at infinity.  The
    sections named in `drop` are masked out entirely."""
    out = dict(sec)
    for k in KEY_POINTS:
        out[k] = bytes(len(sec[k]))
    pts = point_range(n_vars, rank, world)
    for k, size in (("A", 64), ("B1", 64), ("C", 64), ("B2", 128)):
        out[k] = _mask(sec[k], size, [] if k in drop else pts)
    out["H"] = _mask(sec["H"], 64, [] if "H" in drop else column_positions(1 << log_n, rank, world))
    return out


def oracle_partials(c, sec: dict, witness: bytes, rank: int, world: int, threads: int = 8) -> bytes:
    """Rank `rank`'s 388-byte partial (A, B1, C, H, B2, no violated row) by three oracle proofs on masked keys."""
    n_vars, log_n = c.info.n_vars, c.info.domain_log2

    def prove(r, drop):
        return oracle_prove(c, mask_key(sec, n_vars, log_n, rank, world, drop), witness, r, 0, threads=threads)

    p_h = prove(0, ("C",))          # pi_A = A, pi_B = B2, pi_C = H
    p_c = prove(0, ("H",))          # pi_C = C
    p_b1 = prove(1, ("C", "H"))     # pi_C = B1
    return p_h[0:64] + p_b1[192:256] + p_c[192:256] + p_h[192:256] + p_h[64:192] + NO_ROW.to_bytes(4, "little")


def key_points(sec: dict) -> bytes:
    """alpha1, beta1, delta1, beta2, delta2 as zke_shard_combine_raw takes them."""
    return b"".join(sec[k] for k in KEY_POINTS)


def combine_raw(sec: dict, partials: bytes, world: int, rs: bytes):
    """zke_shard_combine_raw: (return code, proof, status, error text)."""
    proof = ctypes.create_string_buffer(256)
    status = ctypes.c_int32(0)
    err = ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_shard_combine_raw(key_points(sec), partials, world, rs, proof, ctypes.byref(status), err, L.ERRCAP)
    return rc, proof.raw, status.value, err.value.decode()


def _rs(r, s):
    return r.to_bytes(32, "little") + s.to_bytes(32, "little")


# --------------------------------------------------------------------------------------------------------------------
LOG_N = 10
R, S = 0x1D2C3B4A59687766554433221100FFEEDDCCBBAA, 0x0F1E2D3C4B5A69788796A5B4C3D2E1F00112233445566


@pytest.fixture(scope="module")
def instance():
    """generate(10) without the heavy bucket (about 800 wires, so the oracle's setup takes a second), its toy key and the
    oracle's unsharded proof at (R, S)."""
    g = generate(LOG_N, seed=5, heavy=False)
    c = z.Circuit.from_r1cs(g["blob"])
    assert c.info.domain_log2 == LOG_N
    sec = oracle_setup(c, (0x1234567, 0x2345, 0x3456, 0x4567, 0x5678))
    want = oracle_prove(c, sec, g["witness"], R, S, threads=4)
    return c, g, sec, want


def test_share_layout_partitions_points_and_columns():
    for n_vars in (1, 7, 803, 1 << 12):
        for world in (2, 4, 8):
            cover = [i for r in range(world) for i in point_range(n_vars, r, world)]
            assert cover == list(range(n_vars))
    for log_n in (6, 10):
        n = 1 << log_n
        for world in (2, 4, 8):
            cols = [column_positions(n, r, world) for r in range(world)]
            assert sorted(np.concatenate(cols).tolist()) == list(range(n))
            for r in range(world):
                assert all(row_owner(int(i), n, world) == r for i in cols[r])
    # G = 4, N = 64: M = 16, four columns of every block
    assert column_positions(64, 1, 4).tolist() == [4, 5, 6, 7, 20, 21, 22, 23, 36, 37, 38, 39, 52, 53, 54, 55]
    with pytest.raises(ValueError):
        column_positions(32, 0, 8)


def test_masked_key_keeps_exactly_the_share(instance):
    c, _, sec, _ = instance
    m, n = c.info.n_vars, 1 << LOG_N
    world, rank = 4, 2
    k = mask_key(sec, m, LOG_N, rank, world)
    for name in KEY_POINTS:
        assert k[name] == bytes(len(sec[name]))
    pts = point_range(m, rank, world)
    for name, size in (("A", 64), ("B1", 64), ("C", 64), ("B2", 128)):
        for i in (0, pts.start - 1, pts.start, pts.stop - 1, pts.stop, m - 1):
            want = sec[name][size * i:size * (i + 1)] if i in pts else bytes(size)
            assert k[name][size * i:size * (i + 1)] == want, (name, i)
    cols = set(column_positions(n, rank, world).tolist())
    for i in range(n):
        assert k["H"][64 * i:64 * (i + 1)] == (sec["H"][64 * i:64 * (i + 1)] if i in cols else bytes(64)), i
    assert mask_key(sec, m, LOG_N, rank, world, ("C", "H"))["C"] == bytes(len(sec["C"]))
    assert sec["A"] != bytes(len(sec["A"]))                       # the original is untouched


@pytest.mark.parametrize("world", [2, 4, 8])
def test_oracle_partials_combine_to_the_unsharded_proof(instance, world):
    c, g, sec, want = instance
    parts = [oracle_partials(c, sec, g["witness"], r, world, threads=4) for r in range(world)]
    assert all(len(p) == L.SHARD_PARTIAL_BYTES for p in parts)
    assert len(set(parts)) == world, "two ranks have the same partial"
    allp = b"".join(parts)
    rc, proof, status, msg = combine_raw(sec, allp, world, _rs(R, S))
    assert (rc, status) == (0, -1), msg
    assert proof == want, "the combined partials differ from the oracle's unsharded proof"
    # a dropped or duplicated share no longer adds up
    rc, proof, _, _ = combine_raw(sec, b"".join(parts[:-1] + parts[:1]), world, _rs(R, S))
    assert rc == 0 and proof != want
    # a flagged row in any one partial: that row is the status, whichever rank saw it; the lowest row wins
    for flagged in range(world):
        bad = bytearray(allp)
        row = 100 + 37 * flagged
        bad[L.SHARD_PARTIAL_BYTES * flagged + 384:L.SHARD_PARTIAL_BYTES * (flagged + 1)] = row.to_bytes(4, "little")
        rc, proof, status, msg = combine_raw(sec, bytes(bad), world, _rs(R, S))
        assert (rc, status) == (1, row) and proof == bytes(256)
        assert msg == f"Assert Failed: constraint {row}"
        if flagged:
            bad[384:388] = (row + 1).to_bytes(4, "little")
            bad[L.SHARD_PARTIAL_BYTES * flagged + 384:L.SHARD_PARTIAL_BYTES * (flagged + 1)] = (row - 1).to_bytes(4, "little")
            assert combine_raw(sec, bytes(bad), world, _rs(R, S))[2] == row - 1
