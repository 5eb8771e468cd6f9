"""Merkle registry of DKIM keys: the tree an app with `"keyRegistryDepth": d` proves its signing key is a leaf of.

A leaf is a key's pubkeyHash - poseidon_large(modulus, ceil(k / 2), 2n), what EmailVerifier outputs - and a node is
H(l, r) = Poseidon(2)([l, r]).  With m leaves and depth d, positions m .. 2^d - 1 hold 0: level l stores ceil(m / 2^l)
nodes, a missing right child at level l is zeros[l] (zeros[0] = 0, zeros[l + 1] = H(zeros[l], zeros[l])), and the root is
level d's single node.  Bit l of a leaf's index is 1 when its ancestor at level l is a right child.  The leaves and the
tree are computed on the GPU (zke_pubkey_hashes, zke_merkle_build), and KeyRegistry.update / append change leaves in
place there (zke_registry_update), rehashing only the ancestors of the changed leaves.

The root says "signed by some key in this set" and nothing about which key, so nothing about which domain: a verifier
compares a proof's registryRoot with the root of the registry it trusts.

A domain-bound registry (build_domains, for specs with `"keyDomain"`) holds (domain, key) pairs instead, as DKIMRegistry's
isDKIMPublicKeyHashValid(domain, pubkeyHash) does: leaf = Poseidon(2)([domain_hash(domain), pubkeyHash]), with
domain_hash = PoseidonModular(PackBytes(domain, 255)) (hash.domain_hash).  Its root says "signed by a key the registry
lists for the domain the proof names".  One key may sit under several domains and one domain may have several keys."""
from __future__ import annotations
import base64
import ctypes
from array import array
import json
import re

from . import _lib as L
from .circuit import FR_MODULUS
from .dkim import parse_tag_list
from .hash import DOMAIN_BYTES, canonical_domain


def _modulus(key) -> int:
    """An RSA modulus from an int or a DKIM TXT record (its `p=` tag, read as dkim.py reads DNS records)."""
    if isinstance(key, int):
        return key
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric import rsa
    tags = parse_tag_list(key.decode() if isinstance(key, bytes) else str(key))
    if not tags.get("p"):
        raise ValueError("DKIM record has no p= tag")
    pub = serialization.load_der_public_key(base64.b64decode(re.sub(r"\s+", "", tags["p"])))
    if not isinstance(pub, rsa.RSAPublicKey):
        raise ValueError("DKIM record does not hold an RSA key")
    return pub.public_numbers().n


def _ints(raw: bytes, count: int) -> list[int]:
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(count)]


def pubkey_hashes(keys, n: int = 121, k: int = 17, device: int = 0) -> list[int]:
    """The pubkeyHash of each key (moduli or DKIM TXT records) on the GPU."""
    moduli = [_modulus(x) for x in keys]
    if not moduli:
        return []
    data, mbytes = _moduli_image(moduli, n, k)
    out = ctypes.create_string_buffer(32 * len(moduli))
    err = ctypes.create_string_buffer(L.ERRCAP)
    if L.zke_pubkey_hashes(data, len(moduli), mbytes, n, k, device, out, err, L.ERRCAP) != 0:
        raise L.ZkeError(err.value.decode())
    return _ints(out.raw, len(moduli))


def _moduli_image(moduli, n: int, k: int) -> tuple[bytes, int]:
    mbytes = max(1, (n * k + 7) // 8, max((m.bit_length() + 7) // 8 for m in moduli))
    return b"".join(m.to_bytes(mbytes, "little") for m in moduli), mbytes


def domain_key_leaves(pairs, n: int = 121, k: int = 17, device: int = 0) -> list[int]:
    """The domain-bound leaf of each (domain, key) pair on the GPU (zke_domain_key_leaves); keys are moduli or DKIM TXT
    records, domains are brought to canonical form (hash.canonical_domain)."""
    pairs = [(canonical_domain(d), _modulus(x)) for d, x in pairs]
    if not pairs:
        return []
    data, mbytes = _moduli_image([m for _, m in pairs], n, k)
    rows = b"".join(d.ljust(DOMAIN_BYTES, b"\0") for d, _ in pairs)
    out = ctypes.create_string_buffer(32 * len(pairs))
    err = ctypes.create_string_buffer(L.ERRCAP)
    if L.zke_domain_key_leaves(data, len(pairs), mbytes, n, k, rows, device, out, err, L.ERRCAP) != 0:
        raise L.ZkeError(err.value.decode())
    return _ints(out.raw, len(pairs))


def domain_key_leaf(domain, key, n: int = 121, k: int = 17) -> int:
    """One domain-bound leaf on the host: Poseidon(2)([domain_hash(domain), pubkeyHash(key)])."""
    from .hash import domain_hash, poseidon, poseidon_large
    return poseidon([domain_hash(domain), poseidon_large(_modulus(key), (k + 1) // 2, 2 * n)])


def merkle_levels(leaves, depth: int, device: int = 0) -> list[list[int]]:
    """Every level of the tree over `leaves` (level 0 = the leaves, the last level = [root]), built on the GPU."""
    leaves = [int(x) for x in leaves]
    err = ctypes.create_string_buffer(L.ERRCAP)
    data = _leaf_image(leaves)
    need = L.zke_merkle_build(data, len(leaves), depth, device, None, 0, err, L.ERRCAP)
    if need < 0:
        raise L.ZkeError(err.value.decode())
    buf = ctypes.create_string_buffer(need)
    if L.zke_merkle_build(data, len(leaves), depth, device, buf, need, err, L.ERRCAP) != need:
        raise L.ZkeError(err.value.decode())
    return _split_levels(buf.raw, len(leaves), depth)


def _leaf_image(leaves) -> bytes:
    """32-byte little-endian leaves; a value outside [0, r) becomes 2^256 - 1, which the library refuses by position."""
    return b"".join(x.to_bytes(32, "little") if 0 <= x < FR_MODULUS else b"\xff" * 32 for x in leaves)


def _split_levels(raw: bytes, count: int, depth: int) -> list[list[int]]:
    """The levels of a tree over `count` leaves from zke_merkle_build's (and zke_registry_levels') flat layout."""
    flat, levels, pos = _ints(raw, len(raw) // 32), [], 0
    for lvl in range(depth + 1):
        size = -(-count // (1 << lvl))
        levels.append(flat[pos:pos + size])
        pos += size
    return levels


def _check_update(changes, count: int, depth: int) -> list[tuple[int, int]]:
    """The (index, leaf) pairs of an update of a tree of `count` leaves and depth `depth`, validated as
    zke_registry_update validates them: each leaf below r (named by its position in the update), no index twice, the
    indices at or above `count` exactly count, count + 1, ... in any order, and at most 2^depth leaves after."""
    pairs = list(changes.items()) if isinstance(changes, dict) else list(changes)
    out = []
    for pos, pair in enumerate(pairs):
        index, leaf = (int(x) for x in pair)
        if index < 0:
            raise ValueError(f"index {index} of the update is negative")
        if not 0 <= leaf < FR_MODULUS:
            raise ValueError(f"leaf {pos} of the update is not below r")
        out.append((index, leaf))
    indices = sorted(i for i, _ in out)
    appended = 0
    for j, i in enumerate(indices):
        if j and i == indices[j - 1]:
            raise ValueError(f"index {i} appears twice")
        if i >= count:
            if i != count + appended:
                raise ValueError(f"index {i} leaves a gap after the {count + appended} leaves")
            appended += 1
    if count + appended > 1 << depth:
        raise ValueError(f"{count + appended} leaves do not fit a tree of depth {depth}")
    return out


class KeyRegistry:
    """A registry of DKIM keys: depth d, the levels of its tree.  build(), build_domains() and from_leaves() compute them on
    the GPU; the constructor only checks shapes.  domain_bound: the leaves are (domain, key) leaves (build_domains).

    update() and append() change leaves in place: on first use they open a copy of the tree resident on `device`
    (zke_registry_open), rehash only the ancestors of the changed leaves there, and patch `levels` with the nodes that
    changed, so root, path, index_of and to_json follow.  Change `levels` only through these methods: the resident tree
    is not read back.  close() (also on garbage collection) frees it; a registry is used by one thread at a time."""

    def __init__(self, depth: int, levels, domain_bound: bool = False, device: int = 0):
        if not isinstance(depth, int) or not 1 <= depth <= 32:
            raise ValueError(f"depth must be 1..32, not {depth!r}")
        levels = [[int(x) for x in lvl] for lvl in levels]
        if len(levels) != depth + 1 or not levels[0] or len(levels[0]) > 1 << depth:
            raise ValueError(f"a tree of depth {depth} has {depth + 1} levels and 1 to 2^{depth} leaves")
        m = len(levels[0])
        for lvl, nodes in enumerate(levels):
            if len(nodes) != -(-m // (1 << lvl)):
                raise ValueError(f"level {lvl} holds {len(nodes)} nodes, not ceil({m} / 2^{lvl})")
        self.depth, self.levels = depth, levels
        self.domain_bound = bool(domain_bound)
        self.device = device
        self._zeros = None
        self._h = None

    @classmethod
    def build(cls, keys, depth: int, n: int = 121, k: int = 17, device: int = 0) -> "KeyRegistry":
        """The registry of `keys` (RSA moduli or DKIM TXT records `v=DKIM1; k=rsa; p=...`), in that order."""
        return cls.from_leaves(pubkey_hashes(keys, n, k, device), depth, device)

    @classmethod
    def build_domains(cls, pairs, depth: int, n: int = 121, k: int = 17, device: int = 0) -> "KeyRegistry":
        """The domain-bound registry of (domain, key) pairs, in that order: what an app spec with "keyDomain" proves
        against.  Domains are lowercased and lose a trailing dot; non-ASCII, empty and over-255-byte names are refused."""
        return cls.from_leaves(domain_key_leaves(pairs, n, k, device), depth, device, domain_bound=True)

    @classmethod
    def from_leaves(cls, leaves, depth: int, device: int = 0, domain_bound: bool = False) -> "KeyRegistry":
        return cls(depth, merkle_levels(leaves, depth, device), domain_bound, device)

    def update(self, changes) -> None:
        """Set leaves: `changes` is a dict or an iterable of (index, leaf) pairs, leaves as field elements (pubkey_hashes,
        domain_key_leaves).  An index below the count replaces that leaf; a leaf of 0 revokes it, and since zeros[0] = 0,
        revoking the last leaves gives the root of the registry without them.  Indices from the count on append and
        must be exactly count, count + 1, ... in any order.  Refused with ValueError, before anything changes: a leaf not
        below r, an index given twice, a gap after the last leaf, more than 2^depth leaves."""
        pairs = _check_update(changes, len(self.levels[0]), self.depth)
        if not pairs:
            return
        h = self._handle()
        err = ctypes.create_string_buffer(L.ERRCAP)
        if L.zke_registry_update(h, array("Q", (i for i, _ in pairs)).tobytes(), b"".join(x.to_bytes(32, "little") for _, x in pairs),
                                 len(pairs), err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
        self._mirror(pairs)

    def append(self, leaves) -> list[int]:
        """Append leaves (field elements) after the last one; returns their indices."""
        first = len(self.levels[0])
        leaves = list(leaves)
        self.update(zip(range(first, first + len(leaves)), leaves))
        return list(range(first, first + len(leaves)))

    def close(self) -> None:
        """Free the resident tree, if one was opened; a later update opens it again from `levels`."""
        h, self._h = getattr(self, "_h", None), None
        if h:
            L.zke_registry_close(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __getstate__(self):
        return dict(self.__dict__, _h=None)        # a copy opens a resident tree of its own

    def _handle(self):
        if self._h is None:
            err = ctypes.create_string_buffer(L.ERRCAP)
            h = L.zke_registry_open(_leaf_image(self.levels[0]), len(self.levels[0]), self.depth, self.device, err, L.ERRCAP)
            if not h:
                raise L.ZkeError(err.value.decode())
            self._h = h
        return self._h

    def _mirror(self, pairs) -> None:
        """Patch `levels` after an update of `pairs` on the device: the ancestors of the changed leaves, fetched with one
        zke_registry_nodes call (new nodes from appends are all among them)."""
        count = max(len(self.levels[0]), max(i for i, _ in pairs) + 1)
        for lvl, nodes in enumerate(self.levels):
            nodes.extend([0] * (-(-count // (1 << lvl)) - len(nodes)))
        for i, x in pairs:
            self.levels[0][i] = x
        changed, lv, ix = sorted(i for i, _ in pairs), [], []
        for lvl in range(1, self.depth + 1):
            changed = sorted({j >> 1 for j in changed})
            lv += [lvl] * len(changed)
            ix += changed
        out, err = ctypes.create_string_buffer(32 * len(ix)), ctypes.create_string_buffer(L.ERRCAP)
        if L.zke_registry_nodes(self._h, array("I", lv).tobytes(), array("Q", ix).tobytes(), len(ix), out, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
        for lvl, j, x in zip(lv, ix, _ints(out.raw, len(ix))):
            self.levels[lvl][j] = x

    @property
    def root(self) -> int:
        return self.levels[-1][0]

    @property
    def leaves(self) -> list[int]:
        return self.levels[0]

    def index_of(self, pubkey_hash: int) -> int:
        """Index of the first leaf equal to pubkey_hash; ValueError if the key is not in the registry."""
        try:
            return self.levels[0].index(int(pubkey_hash))
        except ValueError:
            raise ValueError("the key (its pubkeyHash) is not in the registry") from None

    def zeros(self) -> list[int]:
        if self._zeros is None:
            from .hash import poseidon
            z = [0]
            for _ in range(self.depth):
                z.append(poseidon([z[-1], z[-1]]))
            self._zeros = z
        return self._zeros

    def path(self, i: int) -> tuple[int, list[int]]:
        """(i, siblings): the authentication path of leaf i, from the leaf's sibling up (the circuit's registryIndex and
        registrySiblings)."""
        if not 0 <= i < len(self.levels[0]):
            raise IndexError(f"leaf {i} is not in a registry of {len(self.levels[0])} keys")
        sib, j = [], i
        for lvl in range(self.depth):
            s = j ^ 1
            sib.append(self.levels[lvl][s] if s < len(self.levels[lvl]) else self.zeros()[lvl])
            j >>= 1
        return i, sib

    def to_json(self) -> str:
        """The depth and the leaves (and "leaf": "domainKey" for a domain-bound registry); from_json rebuilds the tree
        on the GPU."""
        d = {"depth": self.depth, "leaves": [str(x) for x in self.levels[0]]}
        if self.domain_bound:
            d["leaf"] = "domainKey"
        return json.dumps(d)

    @classmethod
    def from_json(cls, text: str, device: int = 0) -> "KeyRegistry":
        d = json.loads(text)
        leaf = d.get("leaf", "pubkeyHash")
        if leaf not in ("pubkeyHash", "domainKey"):
            raise ValueError(f'unknown registry leaf {leaf!r}: "pubkeyHash" or "domainKey"')
        return cls.from_leaves([int(x) for x in d["leaves"]], int(d["depth"]), device, domain_bound=leaf == "domainKey")


__all__ = ["KeyRegistry", "pubkey_hashes", "domain_key_leaves", "domain_key_leaf", "merkle_levels"]
