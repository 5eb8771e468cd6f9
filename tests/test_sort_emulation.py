"""Two-level bucket sort of the MSM digits (zk-email-verify_b200/csrc/msm_sort.cuh, DigitSort in msm.cu) checked on the
CPU against a Python counting sort: hist, offsets and the multiset of entries of every bucket (the order inside a bucket
is not fixed).  Cases: uniform digits, every digit in one bucket, empty input, partitions spanning many fine-pass tiles,
bucket counts that are not a multiple of the partition size, and the parameters of the H MSM (2^19 buckets in 256
partitions, 16384-digit tiles)."""
import ctypes
import os
import random
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build():
    out = os.path.join(tempfile.gettempdir(), "libzke_sort_emulation_%d.so" % os.getuid())
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zk-email-verify_b200", "csrc"),
                           os.path.join(ROOT, "tests", "sort_emulation.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    lib.sort_digits.restype = ctypes.c_uint32
    return lib


lib = _build()
U32 = ctypes.c_uint32


def _sort(buckets, n_blocks, n_buckets, fine_bits, tile, rng):
    """digits dealt to n_blocks coarse blocks in order; returns (hist, offsets, entries, words, tiles)"""
    n = len(buckets)
    words = [rng.randrange(1 << 32) for _ in range(n)]
    blocks = sorted(rng.randrange(n_blocks) for _ in range(n))
    arr = lambda xs: (U32 * max(1, len(xs)))(*xs)
    hist, offsets, entries = (U32 * (n_buckets + 1))(), (U32 * (n_buckets + 1))(), (U32 * max(1, n))()
    tiles = lib.sort_digits(arr(buckets), arr(words), arr(blocks), n, n_blocks, n_buckets, fine_bits, tile, hist, offsets, entries)
    return list(hist), list(offsets), list(entries)[:n], words, tiles


def _check(buckets, n_blocks, n_buckets, fine_bits, tile, seed=1):
    hist, offsets, entries, words, tiles = _sort(buckets, n_blocks, n_buckets, fine_bits, tile, random.Random(seed))
    want = [[] for _ in range(n_buckets)]
    for b, w in zip(buckets, words):
        want[b].append(w)
    assert hist[:n_buckets] == [len(x) for x in want] and hist[n_buckets] == 0
    run = 0
    for b in range(n_buckets):
        assert offsets[b] == run, b
        assert sorted(entries[run:run + hist[b]]) == sorted(want[b]), b
        run += hist[b]
    assert offsets[n_buckets] == len(buckets)
    return tiles


def test_uniform_digits():
    rng = random.Random(3)
    for n_buckets, fine_bits, tile in [(1000, 3, 16), (1024, 4, 7), (64, 6, 5), (1 << 19, 11, 16384)]:
        _check([rng.randrange(n_buckets) for _ in range(3000)], 13, n_buckets, fine_bits, tile)


def test_every_digit_in_one_bucket():
    for b in (0, 517, 999):
        tiles = _check([b] * 2000, 9, 1000, 3, 16)
        assert tiles == 2000 // 16    # one partition holds everything, cut into full tiles


def test_empty_input():
    assert _check([], 4, 1000, 3, 16) == 0
    assert _check([], 1, 1 << 19, 11, 16384) == 0


def test_partition_larger_than_a_tile():
    rng = random.Random(5)
    # a few heavy buckets (small witness scalars) beside sparse ones, and empty partitions between them
    buckets = [rng.choice((0, 1, 130)) for _ in range(5000)] + [rng.randrange(256, 512) for _ in range(300)]
    tiles = _check(buckets, 7, 4096, 7, 256)
    assert tiles > 5000 // 256
    # H MSM parameters: one partition of 3 x 16384 + 1 digits
    _check([rng.randrange(2048, 4096) for _ in range(3 * 16384 + 1)] + [rng.randrange(1 << 19) for _ in range(500)], 5, 1 << 19, 11, 16384)
