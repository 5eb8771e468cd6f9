"""Binary Poseidon Merkle tree of the key registry, restated independently of the library.

TEST INFRASTRUCTURE (oracle) - never imported by the product path.

Node H(l, r) = poseidon([l, r]) (oracle/poseidon.py).  With m leaves and depth d, positions m .. 2^d - 1 hold 0; level l
stores ceil(m / 2^l) nodes, a missing right child at level l is zeros[l] (zeros[0] = 0, zeros[l + 1] = H(zeros[l],
zeros[l])); the root is level d's single node.  Bit l of a leaf's index is 1 when its ancestor at level l is a right
child.
"""
from __future__ import annotations

from .poseidon import R, poseidon


def zeros(depth: int) -> list[int]:
    z = [0]
    for _ in range(depth):
        z.append(poseidon([z[-1], z[-1]]))
    return z


def levels(leaves, depth: int) -> list[list[int]]:
    leaves = [int(x) for x in leaves]
    assert 1 <= depth <= 32 and 1 <= len(leaves) <= 1 << depth and all(0 <= x < R for x in leaves)
    z = zeros(depth)
    out = [leaves]
    for lvl in range(depth):
        below = out[-1]
        out.append([poseidon([below[2 * j], below[2 * j + 1] if 2 * j + 1 < len(below) else z[lvl]])
                    for j in range((len(below) + 1) // 2)])
    return out


def root(leaves, depth: int) -> int:
    return levels(leaves, depth)[-1][0]


def path(lv: list[list[int]], index: int) -> list[int]:
    depth = len(lv) - 1
    z = zeros(depth)
    sib = []
    for lvl in range(depth):
        s = (index >> lvl) ^ 1
        sib.append(lv[lvl][s] if s < len(lv[lvl]) else z[lvl])
    return sib


def root_from_path(leaf: int, index: int, siblings) -> int:
    """The root a (leaf, index, siblings) path leads to: at level l, bit l of index puts the node on the right."""
    cur = int(leaf)
    for lvl, s in enumerate(siblings):
        cur = poseidon([int(s), cur] if (index >> lvl) & 1 else [cur, int(s)])
    return cur


def check_path(root_value: int, leaf: int, index: int, siblings) -> bool:
    return 0 <= index < 1 << len(siblings) and root_from_path(leaf, index, siblings) == root_value
