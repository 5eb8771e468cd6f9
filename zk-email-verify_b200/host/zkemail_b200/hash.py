"""Poseidon hashes of the helpers package (packages/helpers/src/hash.ts), on the library's host permutation
(zke_poseidon_hash: circomlib's parameters, the permutation the circuits constrain).

    poseidon(inputs)                                  Poseidon(n) of 1..16 field elements
    poseidon_large(value, num_chunks, bits_per_chunk) poseidonLarge: the little-endian chunks of value, hashed once
    poseidon_modular(inputs)                          poseidonModular: chunks of 16 hashed, the chunk hashes folded left
                                                      to right with Poseidon(2) - the PoseidonModular template
    poseidon_batch(rows, device=0)                    Poseidon of every row (1..16 elements, one width) on the GPU
    domain_hash(domain)                               PoseidonModular(PackBytes(domain, 255)): one Poseidon(9), the
                                                      domain half of a domain-bound registry leaf

Inputs are reduced modulo r as circomlibjs does; outputs are ints below r."""
from __future__ import annotations
import ctypes

from . import _lib as L
from .binary_format import bigint_to_chunked_bytes
from .circuit import FR_MODULUS

CHUNK_SIZE = 16


def poseidon(inputs) -> int:
    """circomlib Poseidon(len(inputs)): state [0, inputs...], output state[0] after the permutation."""
    vals = [int(x) % FR_MODULUS for x in inputs]
    if not 1 <= len(vals) <= CHUNK_SIZE:
        raise ValueError(f"Poseidon takes 1 to {CHUNK_SIZE} inputs, not {len(vals)}")
    out = ctypes.create_string_buffer(32)
    if L.zke_poseidon_hash(b"".join(v.to_bytes(32, "little") for v in vals), len(vals), out) != 0:
        raise L.ZkeError("zke_poseidon_hash failed")
    return int.from_bytes(out.raw, "little")


def poseidon_large(value: int, num_chunks: int, bits_per_chunk: int) -> int:
    """poseidonLarge(input, numChunks, bitsPerChunk): Poseidon of the num_chunks little-endian bits_per_chunk-bit chunks."""
    return poseidon([int(x) for x in bigint_to_chunked_bytes(int(value), bits_per_chunk, num_chunks)])


def poseidon_modular(inputs) -> int:
    """poseidonModular(inputs): what an app circuit's `"reveal": "hash"` output holds for the packed bytes of the part."""
    vals = [int(x) for x in inputs]
    out = None
    for start in range(0, len(vals), CHUNK_SIZE):
        h = poseidon(vals[start:start + CHUNK_SIZE])
        out = h if out is None else poseidon([out, h])
    if out is None:
        raise ValueError("No inputs provided")
    return out


def poseidon_batch(rows, device: int = 0) -> list[int]:
    """[poseidon(row) for row in rows] on the GPU (zke_poseidon_batch): every row has the same width 1..16; values are
    reduced modulo r like poseidon's."""
    rows = [[int(x) % FR_MODULUS for x in r] for r in rows]
    if not rows:
        return []
    width = len(rows[0])
    if not 1 <= width <= CHUNK_SIZE or any(len(r) != width for r in rows):
        raise ValueError(f"every row needs the same width of 1 to {CHUNK_SIZE} inputs")
    data = b"".join(v.to_bytes(32, "little") for r in rows for v in r)
    out = ctypes.create_string_buffer(32 * len(rows))
    err = ctypes.create_string_buffer(L.ERRCAP)
    if L.zke_poseidon_batch(data, width, len(rows), device, out, err, L.ERRCAP) != 0:
        raise L.ZkeError(err.value.decode())
    raw = out.raw
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(len(rows))]


DOMAIN_BYTES = 255           # a DNS name has at most 255 bytes: PackBytes(D, 255) is 9 words


def canonical_domain(domain) -> bytes:
    """The canonical form of a domain name: ASCII (an international name in its A-label form, xn--...), lower case,
    without a trailing dot, 1..255 bytes and no zero byte.  Lowercases and strips one trailing dot; ValueError otherwise."""
    if isinstance(domain, str):
        try:
            raw = domain.encode("ascii")
        except UnicodeEncodeError:
            raise ValueError(f"domain {domain!r} is not ASCII: give an international name in its A-label (xn--) form") from None
    else:
        raw = bytes(domain)
        if any(c >= 0x80 for c in raw):
            raise ValueError(f"domain {raw!r} is not ASCII: give an international name in its A-label (xn--) form")
    raw = raw.lower()
    if raw.endswith(b"."):
        raw = raw[:-1]
    if not 1 <= len(raw) <= DOMAIN_BYTES:
        raise ValueError(f"domain {raw!r} has {len(raw)} bytes; a domain has 1 to {DOMAIN_BYTES}")
    if 0 in raw:
        raise ValueError(f"domain {raw!r} holds a zero byte")
    return raw


def domain_words(raw: bytes) -> list[int]:
    """PackBytes(raw, 255): the 9 little-endian 31-byte words of the zero-padded name (no canonical check)."""
    raw = raw.ljust(DOMAIN_BYTES, b"\0")
    return [int.from_bytes(raw[31 * i:31 * i + 31], "little") for i in range(9)]


def domain_hash(domain) -> int:
    """PoseidonModular(PackBytes(canonical_domain(domain), 255)), one Poseidon(9): what a `"reveal": "hash"` part of
    maxLength 255 publishes for the name, whatever maxLength the part that binds the registry leaf has."""
    return poseidon(domain_words(canonical_domain(domain)))


__all__ = ["poseidon", "poseidon_large", "poseidon_modular", "poseidon_batch", "canonical_domain", "domain_hash"]
