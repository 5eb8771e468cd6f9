"""In-place registry updates without a GPU: the ABI symbols, zke_registry_open's refusals (those of zke_merkle_build,
word for word), KeyRegistry.update / append refusing a duplicate, a gap, an overflow past 2^depth and a leaf not below r
before anything changes, and revocation (a leaf set to 0) of the last leaves giving the tree without them, on the
oracle."""
import ctypes
import random

import pytest

import zkemail_b200 as z
from oracle import merkle

R = z.FR_MODULUS
L = z._lib

SYMBOLS = ["zke_registry_open", "zke_registry_update", "zke_registry_nodes", "zke_registry_levels", "zke_registry_count",
           "zke_registry_close"]


def test_symbols_present():
    for name in SYMBOLS:
        assert hasattr(L.lib, name), name


@pytest.mark.parametrize("count,depth", [(1, 0), (1, 33), (0, 10), (1025, 10), (3, 1)])
def test_open_refuses_what_merkle_build_refuses(count, depth):
    """Each refusal comes before a device is touched, with zke_merkle_build's message."""
    leaves = bytes(32 * max(count, 1))
    err_open, err_build = ctypes.create_string_buffer(L.ERRCAP), ctypes.create_string_buffer(L.ERRCAP)
    assert not L.zke_registry_open(leaves, count, depth, 0, err_open, L.ERRCAP)
    assert L.zke_merkle_build(leaves, count, depth, 0, None, 0, err_build, L.ERRCAP) < 0
    assert err_open.value and err_open.value == err_build.value
    assert not L.zke_registry_open(None, 1, 10, 0, err_open, L.ERRCAP)
    assert err_open.value == b"null argument"


def test_null_handle_is_refused():
    err = ctypes.create_string_buffer(L.ERRCAP)
    assert L.zke_registry_update(None, bytes(8), bytes(32), 1, err, L.ERRCAP) < 0 and err.value == b"null registry"
    assert L.zke_registry_nodes(None, bytes(4), bytes(8), 1, ctypes.create_string_buffer(32), err, L.ERRCAP) < 0
    assert L.zke_registry_levels(None, None, 0, err, L.ERRCAP) < 0 and err.value == b"null registry"
    assert L.zke_registry_count(None) == 0
    L.zke_registry_close(None)


def _registry(count, depth, seed=1):
    rng = random.Random(seed)
    return z.KeyRegistry(depth, merkle.levels([rng.randrange(R) for _ in range(count)], depth))


@pytest.fixture(scope="module")
def small():
    return _registry(10, 10)


@pytest.mark.parametrize("changes,message", [
    ([(7, 1), (3, 2), (7, 3)], "index 7 appears twice"),
    ({12: 5}, "index 12 leaves a gap after the 10 leaves"),
    ([(10, 1), (12, 2), (3, 4)], "index 12 leaves a gap after the 11 leaves"),
    ([(0, 1), (3, R)], "leaf 1 of the update is not below r"),
    ([(0, -1)], "leaf 0 of the update is not below r"),
    ([(-1, 1)], "index -1 of the update is negative"),
])
def test_update_refusals(small, changes, message):
    before = [list(x) for x in small.levels]
    with pytest.raises(ValueError, match=message):
        small.update(changes)
    assert small.levels == before and small._h is None          # refused on the host, nothing opened


def test_append_refuses_overflow():
    reg = _registry(1020, 10)
    before = [list(x) for x in reg.levels]
    with pytest.raises(ValueError, match="^1025 leaves do not fit a tree of depth 10$"):
        reg.append([1, 2, 3, 4, 5])
    with pytest.raises(ValueError, match="^17 leaves do not fit a tree of depth 4$"):
        _registry(16, 4).append([0])
    assert reg.levels == before and reg._h is None


def test_empty_update_does_nothing(small):
    before = [list(x) for x in small.levels]
    small.update({})
    assert small.append([]) == []
    assert small.levels == before and small._h is None


@pytest.mark.parametrize("depth,count", [(1, 2), (4, 11), (10, 300)])
def test_revoking_the_last_leaves_equals_removing_them(depth, count):
    """Revoked leaves are 0 = zeros[0]: every node that covers only revoked leaves equals zeros[l], every other node is
    the node of the tree without them, and the roots are equal."""
    rng = random.Random(depth)
    leaves = [rng.randrange(1, R) for _ in range(count)]
    zeros = merkle.zeros(depth)
    for gone in sorted({1, count // 2, count - 1}):
        kept = leaves[:count - gone]
        revoked = merkle.levels(kept + [0] * gone, depth)
        removed = merkle.levels(kept, depth)
        assert revoked[-1][0] == removed[-1][0]
        for lvl in range(depth + 1):
            n = len(removed[lvl])
            assert revoked[lvl][:n] == removed[lvl]
            assert revoked[lvl][n:] == [zeros[lvl]] * (len(revoked[lvl]) - n)
        assert revoked[-1][0] != merkle.root(leaves, depth)
