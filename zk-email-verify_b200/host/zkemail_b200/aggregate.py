"""Aggregation of n Groth16 proofs under one key into one O(log n) proof (SnarkPack; DESIGN.md "Proof aggregation").

    srs = AggSrs.from_ptau(ptau_a, ptau_b, n_max)      # two Powers-of-Tau files with independent taus
    agg = aggregate(srs, vkey, proofs, publics)        # GPU prover; a JSON-able dict
    verify_aggregate(srs.vk(), vkey, publics, agg)      # host verifier: O(log n) pairings

`proofs` are snarkjs proof objects or one bytes object in zke_prove's layout ([n][8][32], the output of Context.prove);
`publics` are per-proof lists of public signals, or bytes in zke_prove's layout ([n][nPublic][32]).
"""
from __future__ import annotations

import ctypes
import json

from . import _lib as L
from .engine import _dec, _g1_bytes, _g2_bytes

_FR = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def _proof_bytes(proofs) -> bytes:
    if isinstance(proofs, (bytes, bytearray, memoryview)):
        return bytes(proofs)
    return b"".join(_g1_bytes(p["pi_a"]) + _g2_bytes(p["pi_b"]) + _g1_bytes(p["pi_c"]) for p in proofs)


def _public_bytes(publics, n_public: int) -> tuple[bytes, int]:
    if isinstance(publics, (bytes, bytearray, memoryview)):
        if n_public == 0 or len(publics) % (32 * n_public):
            raise L.ZkeError("public-signal bytes are not a whole number of proofs")
        return bytes(publics), len(publics) // (32 * n_public)
    out = b""
    for i, row in enumerate(publics):
        if len(row) != n_public:
            raise L.ZkeError(f"proof {i} has {len(row)} public signals, the key expects {n_public}")
        for s in row:
            x = _dec(s)
            if x >= _FR:
                raise L.ZkeError("public signal not below r")
            out += x.to_bytes(32, "little")
    return out, len(publics)


class AggSrs:
    """The prover's SRS on GPU `device`: h^(a^i), h^(b^i) for i < n_max and g^(a^i), g^(b^i) for i < 2 n_max, read from two
    `.ptau` files (their tauG2 / tauG1 sections) whose points are checked on the device."""

    def __init__(self, handle, n_max: int, device: int):
        self._h, self.n_max, self.device = handle, n_max, device

    @classmethod
    def from_ptau(cls, ptau_a, ptau_b, n_max: int, device: int = 0) -> "AggSrs":
        err = ctypes.create_string_buffer(L.ERRCAP)
        a, b = bytes(ptau_a), bytes(ptau_b)
        h = L.zke_agg_srs_from_ptau(a, len(a), b, len(b), n_max, device, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return cls(h, n_max, device)

    def vk(self) -> dict:
        """The verifier key {g, h, g_a, g_b, h_a, h_b} (snarkjs point encoding)."""
        n = ctypes.c_size_t(0)
        L.zke_agg_vk_json(self._h, None, ctypes.byref(n))
        buf = ctypes.create_string_buffer(n.value)
        if L.zke_agg_vk_json(self._h, buf, ctypes.byref(n)) != 0:
            raise L.ZkeError("zke_agg_vk_json failed")
        return json.loads(buf.value.decode())

    def close(self):
        if getattr(self, "_h", None):
            L.zke_agg_srs_free(self._h)
            self._h = None

    __del__ = close


def aggregate_raw(srs: AggSrs, vkey: dict, proofs256: bytes, publics: bytes, n: int) -> bytes:
    size = L.zke_agg_bytes(n)
    out = ctypes.create_string_buffer(max(size, 1))
    err = ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_aggregate(srs._h, json.dumps(vkey).encode(), n, bytes(proofs256), bytes(publics) if publics else None, out,
                         size, err, L.ERRCAP)
    if rc < 0:
        raise L.ZkeError(err.value.decode())
    return out.raw[:rc]


def aggregate(srs: AggSrs, vkey: dict, proofs, publics) -> dict:
    """n proofs under `vkey` (n a power of two from 2 to 8192, at most srs.n_max) -> {"protocol", "curve", "n", "aggregate":
    hex of the aggregate's bytes}."""
    pb = _proof_bytes(proofs)
    sb, n = _public_bytes(publics, len(vkey["IC"]) - 1) if len(vkey["IC"]) > 1 else (b"", len(pb) // 256)
    if len(pb) != 256 * n:
        raise L.ZkeError(f"{len(pb) // 256} proofs for {n} public-signal vectors")
    return {"protocol": "snarkpack", "curve": "bn128", "n": n, "aggregate": aggregate_raw(srs, vkey, pb, sb, n).hex()}


def verify_aggregate(agg_vk: dict, vkey: dict, publics, agg) -> bool:
    """True iff `agg` (a dict from aggregate(), or its bytes) proves valid proofs under `vkey` for these public signals.
    Raises ZkeError on malformed input: a count that is not a power of two, wrong lengths, points off their curves."""
    data = bytes.fromhex(agg["aggregate"]) if isinstance(agg, dict) else bytes(agg)
    n_public = len(vkey["IC"]) - 1
    sb, n = _public_bytes(publics, n_public) if n_public else (b"", int(agg["n"]) if isinstance(agg, dict) else 0)
    if isinstance(agg, dict) and int(agg["n"]) != n:
        raise L.ZkeError(f"the aggregate is of {agg['n']} proofs, not {n}")
    err = ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_agg_verify(json.dumps(agg_vk).encode(), json.dumps(vkey).encode(), n, sb if sb else None, data, len(data), err,
                          L.ERRCAP)
    if rc < 0:
        raise L.ZkeError(err.value.decode())
    return rc == 1
