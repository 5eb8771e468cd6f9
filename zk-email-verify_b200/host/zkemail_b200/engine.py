"""Proving key and GPU context wrappers over the C ABI (zke_setup / zke_ctx_* / zke_witness / zke_prove)."""
from __future__ import annotations
import ctypes
import json
from . import _lib as L
from ._mapped import mapped_buffer
from .circuit import Circuit


class AssertFailed(L.ZkeError):
    """Raised when a witness violates a constraint; the message contains "Assert Failed" - the string the
    reference's tests match (/root/reference/packages/circuits/tests/email-verifier.test.ts:78)."""


def device_count() -> int:
    return L.zke_device_count()


class Zkey:
    """Groth16 proving key resident on one GPU.  `Zkey(circuit, seed)` runs the TOY seeded setup (known toxic waste:
    tests and benchmarks only); `Zkey.load(bytes)` / `Zkey.load_chunks([...])` ingest a real snarkjs `.zkey`."""

    def __init__(self, circuit: Circuit | None, seed: int = 1, device: int = 0, _handle=None):
        if _handle is None:
            err = ctypes.create_string_buffer(L.ERRCAP)
            _handle = L.zke_setup(circuit.handle, seed, device, err, L.ERRCAP)
            if not _handle:
                raise L.ZkeError(err.value.decode())
        self._h = _handle
        self.circuit, self.device = circuit, device

    @classmethod
    def load(cls, zkey_bytes: bytes, device: int = 0, circuit: Circuit | None = None):
        """`${circuitName}.zkey` as handed to snarkjs.groth16.fullProve (chunked-zkey.ts:80-84)."""
        err = ctypes.create_string_buffer(L.ERRCAP)
        h = L.zke_zkey_load(zkey_bytes, len(zkey_bytes), device, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return cls(circuit, device=device, _handle=h)

    @classmethod
    def load_chunks(cls, chunks, device: int = 0, circuit: Circuit | None = None):
        """The fork's chunked key: chunks[i] = contents of `${circuitName}.zkey{b..k}[i]` (chunked-zkey.ts:9,35-37)."""
        keep = [bytes(c) for c in chunks]
        ptrs = (L.c_void_p * len(keep))(*[ctypes.cast(ctypes.c_char_p(c), L.c_void_p) for c in keep])
        lens = (L.c_size_t * len(keep))(*[len(c) for c in keep])
        err = ctypes.create_string_buffer(L.ERRCAP)
        h = L.zke_zkey_load_chunks(ptrs, lens, len(keep), device, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return cls(circuit, device=device, _handle=h)

    @classmethod
    def from_ptau(cls, circuit: Circuit, ptau, device: int = 0):
        """`snarkjs groth16 setup` for this engine's R1CS: a key from a prepared phase-2 `.ptau` (bytes, a writable buffer or
        a path, which is memory-mapped).  gamma = delta = 1, so the key is a toy until `contribute` is applied."""
        err = ctypes.create_string_buffer(L.ERRCAP)
        with mapped_buffer(ptau) as (ptr, n):
            h = L.zke_zkey_from_ptau(circuit.handle, ptr, n, device, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return cls(circuit, device=device, _handle=h)

    def contribute(self, secret: bytes | None = None) -> "Zkey":
        """Phase-2 contribution (`snarkjs zkey contribute`, without its transcript): a new key with delta times s and the L
        and H points times 1/s.  secret: 32 bytes LE in (1, r); None draws it from `secrets`.  The secret is not kept."""
        if secret is None:
            import secrets
            from .circuit import FR_MODULUS
            secret = (secrets.randbelow(FR_MODULUS - 2) + 2).to_bytes(32, "little")
        if len(secret) != 32:
            raise ValueError("secret must be 32 bytes")
        err = ctypes.create_string_buffer(L.ERRCAP)
        h = L.zke_zkey_contribute(self._h, bytes(secret), err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return Zkey(self.circuit, device=self.device, _handle=h)

    def contribution_report(self, prev: "Zkey", rand: bytes | None = None) -> tuple[bool, str]:
        """(True, "") if this key follows from `prev` by phase-2 contributions, else (False, reason): the ratio check of
        `snarkjs zkey verify`.  rand: 16 bytes that seed the random weights (default: drawn by the library)."""
        if rand is not None and len(rand) != 16:
            raise ValueError("rand must be 16 bytes")
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_zkey_check_contribution(prev._h, self._h, bytes(rand) if rand is not None else None, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        return rc == 1, err.value.decode()

    def check_contribution(self, prev: "Zkey", rand: bytes | None = None) -> bool:
        return self.contribution_report(prev, rand)[0]

    @property
    def is_toy(self) -> bool:
        return L.zke_zkey_is_toy(self._h) == 1

    @property
    def info(self):
        a, b, c = L.c_u32(), L.c_u32(), L.c_u32()
        L.zke_zkey_info(self._h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        return {"n_vars": a.value, "n_public": b.value, "domain_log2": c.value}

    def write(self) -> bytes:
        """The key as a `.zkey` file image (iden3 binfile, what `snarkjs groth16 setup` writes)."""
        ch = self.circuit.handle if self.circuit is not None else None
        n = L.zke_zkey_write(self._h, ch, None, 0)
        if n < 0:
            raise L.ZkeError("zkey export failed (a key made by the toy setup needs its circuit)")
        buf = ctypes.create_string_buffer(n)
        if L.zke_zkey_write(self._h, ch, buf, n) != n:
            raise L.ZkeError("zkey export failed")
        return buf.raw

    def __del__(self):
        if getattr(self, "_h", None):
            L.zke_zkey_free(self._h)
            self._h = None

    @property
    def handle(self):
        return self._h

    def vkey(self) -> dict:
        """`snarkjs zkey export verificationkey` -> vkey.json object."""
        n = L.c_size_t(0)
        L.zke_zkey_vkey_json(self._h, None, ctypes.byref(n))
        buf = ctypes.create_string_buffer(n.value)
        n2 = L.c_size_t(n.value)
        if L.zke_zkey_vkey_json(self._h, buf, ctypes.byref(n2)) != 0:
            raise L.ZkeError("vkey export failed")
        return json.loads(buf.value.decode())

    def section(self, sec: int) -> bytes:
        cnt = L.zke_zkey_section(self._h, sec, None, 0)
        if cnt < 0:
            raise L.ZkeError("bad section")
        size = 128 if sec in (L.SEC_BETA2, L.SEC_GAMMA2, L.SEC_DELTA2, L.SEC_B2) else 64
        buf = ctypes.create_string_buffer(size * cnt)
        if L.zke_zkey_section(self._h, sec, buf, len(buf)) < 0:
            raise L.ZkeError("section read failed")
        return buf.raw



def ptau_info(ptau, circuit: Circuit | None = None) -> dict:
    """Structure of a prepared `.ptau` as the library reads it (host only): {"power", "sections": {type: (offset, size)}}.
    Raises ZkeError with the library's message for a malformed file or one too small for `circuit`."""
    power = L.c_u32()
    offs, sizes = (L.c_u64 * 16)(), (L.c_u64 * 16)()
    err = ctypes.create_string_buffer(L.ERRCAP)
    with mapped_buffer(ptau) as (ptr, n):
        rc = L.zke_ptau_info(circuit.handle if circuit is not None else None, ptr, n, ctypes.byref(power), offs, sizes, err, L.ERRCAP)
    if rc != 0:
        raise L.ZkeError(err.value.decode())
    return {"power": power.value, "sections": {s: (offs[s], sizes[s]) for s in range(16) if sizes[s] or offs[s]}}


def ptau_toy(power: int, tau: int, alpha: int, beta: int, device: int = 0) -> bytearray:
    """TOY prepared `.ptau` from KNOWN (tau, alpha, beta): tests and measurement only (anyone holding it can forge)."""
    tab = b"".join(int(v).to_bytes(32, "little") for v in (tau, alpha, beta))
    err = ctypes.create_string_buffer(L.ERRCAP)
    n = L.zke_ptau_toy(power, tab, device, None, 0, err, L.ERRCAP)
    if n < 0:
        raise L.ZkeError(err.value.decode())
    out = bytearray(n)
    arr = (ctypes.c_char * n).from_buffer(out)
    got = L.zke_ptau_toy(power, tab, device, ctypes.cast(arr, L.c_void_p), n, err, L.ERRCAP)
    del arr
    if got != n:
        raise L.ZkeError(err.value.decode() or "ptau writer failed")
    return out


def _ptau_write(call) -> bytearray:
    """Runs a `.ptau` writer of the C ABI twice: for its size (out = NULL), then into a new bytearray."""
    err = ctypes.create_string_buffer(L.ERRCAP)
    n = call(None, 0, err)
    if n < 0:
        raise L.ZkeError(err.value.decode())
    out = bytearray(n)
    arr = (ctypes.c_char * n).from_buffer(out)
    got = call(ctypes.cast(arr, L.c_void_p), n, err)
    del arr
    if got != n:
        raise L.ZkeError(err.value.decode() or "ptau writer failed")
    return out


def ptau_new(power: int) -> bytearray:
    """`snarkjs powersoftau new`: an unprepared `.ptau` (sections 1-7) of `power` whose points are all the generators."""
    return _ptau_write(lambda out, cap, err: L.zke_ptau_new(power, out, cap, err, L.ERRCAP))


def ptau_contribute(ptau, secrets: tuple | None = None, device: int = 0) -> tuple[bytearray, bytes]:
    """`snarkjs powersoftau contribute` (without its transcript): (new unprepared `.ptau`, receipt).  secrets: (tau, alpha,
    beta) ints in [2, r); None draws them from the OS.  The receipt, [tau]_2 | [alpha]_2 | [beta]_2 (384 bytes), is the
    public part of the contribution: verify_ptau(new, prev=ptau, receipt=receipt) checks that `new` builds on `ptau`."""
    tab = None if secrets is None else b"".join(int(v).to_bytes(32, "little") for v in secrets)
    if tab is not None and len(tab) != 96:
        raise ValueError("secrets must be three integers below 2^256")
    receipt = ctypes.create_string_buffer(384)
    with mapped_buffer(ptau) as (ptr, n):
        out = _ptau_write(lambda o, cap, err: L.zke_ptau_contribute(ptr, n, tab, device, o, cap, receipt if o else None, err, L.ERRCAP))
    return out, receipt.raw


def ptau_prepare(ptau, device: int = 0) -> bytearray:
    """`snarkjs powersoftau prepare phase2`: the unprepared `.ptau` plus its Lagrange sections 12-15, computed on the GPU."""
    with mapped_buffer(ptau) as (ptr, n):
        return _ptau_write(lambda out, cap, err: L.zke_ptau_prepare(ptr, n, device, out, cap, err, L.ERRCAP))


def ptau_report(ptau, prev=None, receipt: bytes | None = None, device: int = 0, rand: bytes | None = None) -> tuple[bool, str]:
    """(True, "") if `ptau` (unprepared or prepared) passes the algebraic checks of `snarkjs powersoftau verify`, else
    (False, reason): valid points, generators at index 0, consecutive powers of one tau in every family, the Lagrange
    sections (if present) the bases of those powers and, with `prev` and `receipt` (both or neither), that `ptau` is `prev`
    after the contribution the receipt describes.  rand: 16 bytes that seed the random weights (default: the library's)."""
    if (prev is None) != (receipt is None):
        raise ValueError("prev and receipt go together")
    if receipt is not None and len(receipt) != 384:
        raise ValueError("receipt must be 384 bytes")
    if rand is not None and len(rand) != 16:
        raise ValueError("rand must be 16 bytes")
    err = ctypes.create_string_buffer(L.ERRCAP)
    with mapped_buffer(ptau) as (ptr, n):
        if prev is None:
            rc = L.zke_ptau_verify(ptr, n, None, 0, None, bytes(rand) if rand is not None else None, device, err, L.ERRCAP)
        else:
            with mapped_buffer(prev) as (pptr, pn):
                rc = L.zke_ptau_verify(ptr, n, pptr, pn, bytes(receipt), bytes(rand) if rand is not None else None, device, err, L.ERRCAP)
    if rc < 0:
        raise L.ZkeError(err.value.decode())
    return rc == 1, err.value.decode()


def verify_ptau(ptau, prev=None, receipt: bytes | None = None, device: int = 0, rand: bytes | None = None) -> bool:
    return ptau_report(ptau, prev, receipt, device, rand)[0]


def verify_zkey(circuit: Circuit, ptau, zkey: Zkey, device: int | None = None, rand: bytes | None = None) -> bool:
    """Whether `zkey` was set up for `circuit` from `ptau` (Zkey.from_ptau) followed by any number of contributions: the
    whole delta chain collapses into one ratio, checked by Zkey.check_contribution."""
    base = Zkey.from_ptau(circuit, ptau, device=zkey.device if device is None else device)
    return zkey.check_contribution(base, rand)


class Context:
    def __init__(self, circuit: Circuit | None, zkey: Zkey | None = None, device: int = 0, max_batch: int = 1):
        err = ctypes.create_string_buffer(L.ERRCAP)
        self._h = L.zke_ctx_open(circuit.handle if circuit is not None else None, zkey.handle if zkey else None, device,
                                 max_batch, err, L.ERRCAP)
        if not self._h:
            raise L.ZkeError(err.value.decode())
        self.circuit, self.zkey, self.device, self.max_batch = circuit, zkey, device, max_batch
        self._pending = []
        self.n_vars = circuit.info.n_vars if circuit is not None else zkey.info["n_vars"]
        self.n_public = circuit.info.n_public if circuit is not None else zkey.info["n_public"]

    def close(self):
        if getattr(self, "_h", None):
            L.zke_ctx_close(self._h)
            self._h = None

    __del__ = close

    @property
    def handle(self):
        return self._h

    @property
    def stream(self) -> int:
        return L.zke_ctx_stream(self._h) or 0

    def upload_inputs(self, packed_inputs, batch: int):
        err = ctypes.create_string_buffer(L.ERRCAP)
        if L.zke_upload_inputs(self._h, packed_inputs, batch, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())

    def profile(self, enable: bool = True):
        L.zke_ctx_profile(self._h, 1 if enable else 0)

    def profile_get(self) -> dict:
        n = len(L.STAGES)
        ms, cnt = (ctypes.c_double * n)(), (L.c_u64 * n)()
        L.zke_ctx_profile_get(self._h, ms, cnt)
        return {name: {"ms": ms[i], "count": cnt[i]} for i, name in enumerate(L.STAGES)}

    def witness(self, packed_inputs, batch: int, want_witness: bool = True, raise_on_fail: bool = True):
        """calculateWitness + checkConstraints.  Returns (witness bytes | None, status list)."""
        m = self.n_vars
        out = ctypes.create_string_buffer(32 * m * batch) if want_witness else None
        status = (ctypes.c_int32 * batch)()
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_witness(self._h, packed_inputs, batch, out, status, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        if rc > 0 and raise_on_fail:
            raise AssertFailed(err.value.decode())
        return (out.raw if out is not None else None), list(status)

    def load_witness(self, wtns: bytes, batch: int):
        err = ctypes.create_string_buffer(L.ERRCAP)
        if L.zke_load_witness(self._h, wtns, batch, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())

    def check_witness(self, batch: int, raise_on_fail: bool = True) -> list:
        """`snarkjs wtns check` for the first `batch` witnesses of load_witness: per witness -1, or the first violated
        constraint.  Raises AssertFailed ("Assert Failed: constraint i ...") when one fails, unless raise_on_fail is False."""
        status = (ctypes.c_int32 * batch)()
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_check_witness(self._h, batch, status, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        if rc > 0 and raise_on_fail:
            raise AssertFailed(err.value.decode())
        return list(status)

    def check_wtns(self, wtns_file: bytes, raise_on_fail: bool = True) -> int:
        """`snarkjs wtns check circuit.r1cs witness.wtns`: one `.wtns` file image against the circuit's constraints.  Returns
        -1 when every constraint holds, else the first violated one (AssertFailed unless raise_on_fail is False)."""
        from .iden3_binfile import read_wtns
        data = read_wtns(bytes(wtns_file))
        if len(data) != 32 * self.n_vars:
            raise L.ZkeError(f".wtns has {len(data) // 32} values, the circuit has {self.n_vars} wires")
        self.load_witness(data, 1)
        return self.check_witness(1, raise_on_fail)[0]

    def _prove_call(self, fn, head_args, batch, rs, raise_on_fail):
        npub = self.n_public
        proofs = ctypes.create_string_buffer(256 * batch)
        publics = ctypes.create_string_buffer(max(1, 32 * npub * batch))
        status = (ctypes.c_int32 * batch)()
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = fn(self._h, *head_args, batch, rs, proofs, publics, status, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        if rc > 0 and raise_on_fail:
            raise AssertFailed(err.value.decode())
        return proofs.raw, publics.raw[: 32 * npub * batch], list(status)

    def prove(self, batch: int, rs: bytes | None = None, raise_on_fail: bool = True):
        return self._prove_call(L.zke_prove, (), batch, rs, raise_on_fail)

    def wtns_prove(self, wtns_file: bytes, rs: bytes | None = None):
        """`snarkjs groth16 prove zkey wtns`: one `.wtns` file image -> (proof bytes, public signal bytes)."""
        npub = self.n_public
        proof = ctypes.create_string_buffer(256)
        publics = ctypes.create_string_buffer(max(1, 32 * npub))
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_wtns_prove(self._h, wtns_file, len(wtns_file), rs, proof, publics, err, L.ERRCAP)
        if rc != 0:
            raise L.ZkeError(err.value.decode())
        return proof.raw, publics.raw[: 32 * npub]

    def submit(self, packed_inputs, batch: int, rs: bytes | None = None):
        """Pipelined fullprove: enqueue one batch (at most two in flight); pair with collect()."""
        err = ctypes.create_string_buffer(L.ERRCAP)
        if L.zke_fullprove_submit(self._h, packed_inputs, batch, rs, err, L.ERRCAP) != 0:
            raise L.ZkeError(err.value.decode())
        self._pending.append(batch)

    def collect(self, raise_on_fail: bool = True):
        batch = self._pending.pop(0)
        npub = self.n_public
        proofs = ctypes.create_string_buffer(256 * batch)
        publics = ctypes.create_string_buffer(max(1, 32 * npub * batch))
        status = (ctypes.c_int32 * batch)()
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_fullprove_collect(self._h, proofs, publics, status, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        if rc > 0 and raise_on_fail:
            raise AssertFailed(err.value.decode())
        return proofs.raw, publics.raw[: 32 * npub * batch], list(status)

    def fullprove(self, packed_inputs, batch: int, rs: bytes | None = None, raise_on_fail: bool = True):
        npub = self.n_public
        proofs = ctypes.create_string_buffer(256 * batch)
        publics = ctypes.create_string_buffer(max(1, 32 * npub * batch))
        status = (ctypes.c_int32 * batch)()
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_fullprove(self._h, packed_inputs, batch, rs, proofs, publics, status, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        if rc > 0 and raise_on_fail:
            raise AssertFailed(err.value.decode())
        return proofs.raw, publics.raw[: 32 * npub * batch], list(status)


def proof_to_json(proof256: bytes, publics: bytes, n_public: int):
    """256-byte proof + packed public signals -> (proof.json object, publicSignals list) in snarkjs format."""
    pl, sl = L.c_size_t(4096), L.c_size_t(80 * max(1, n_public) + 16)
    pj, sj = ctypes.create_string_buffer(pl.value), ctypes.create_string_buffer(sl.value)
    if L.zke_proof_to_json(proof256, publics, n_public, pj, ctypes.byref(pl), sj, ctypes.byref(sl)) != 0:
        raise L.ZkeError("proof_to_json failed")
    return json.loads(pj.value.decode()), json.loads(sj.value.decode())


def verify_batch(vkey: dict, public_signals_list, proofs, rand: bytes | None = None) -> list:
    """n proofs under one verification key with ONE randomised product of pairings (n + 3 Miller loops, one final
    exponentiation) - SURVEY 8(f) rank 4; per-proof verdicts, identical to [verify(vkey, s, p) for ...] (a false proof slips
    through with probability ~2^-128 over `rand`, 16 fresh bytes per proof; default os.urandom)."""
    import os
    n = len(proofs)
    if len(public_signals_list) != n:
        raise ValueError("one public-signal list per proof")
    if n == 0:
        return []
    rand = os.urandom(16 * n) if rand is None else rand
    if len(rand) != 16 * n:
        raise ValueError("rand must hold 16 bytes per proof")
    err = ctypes.create_string_buffer(L.ERRCAP)
    ok = ctypes.create_string_buffer(n)
    rbuf = ctypes.create_string_buffer(bytes(rand), 16 * n)
    rc = L.zke_verify_batch_json(json.dumps(vkey).encode(),
                                 json.dumps([[str(s) for s in sig] for sig in public_signals_list]).encode(),
                                 json.dumps(list(proofs)).encode(), ctypes.cast(rbuf, ctypes.c_void_p), ctypes.cast(ok, ctypes.c_void_p),
                                 err, L.ERRCAP)
    if rc < 0:
        raise L.ZkeError(err.value.decode())
    return [b == 1 for b in ok.raw]


_FQ = 21888242871839275222246405745257275088696311157297823662689037894645226208583
_OFF_CURVE_A = (1).to_bytes(32, "little") * 2       # (1, 1) is not on y^2 = x^3 + 3


def _dec(v) -> int:
    """A decimal string or number as zke_verify_batch_json reads it (the same errors for malformed values)."""
    s = v if isinstance(v, str) else str(v)
    if not s or not s.isascii() or not s.isdigit():
        raise L.ZkeError("expected a decimal string")
    x = int(s)
    if x >> 256:
        raise L.ZkeError("decimal value does not fit 256 bits")
    return x


def _fq_bytes(v) -> bytes:
    x = _dec(v)
    if x >= _FQ:
        raise L.ZkeError("coordinate not reduced")
    return x.to_bytes(32, "little")


def _g1_bytes(v) -> bytes:
    if not isinstance(v, list) or len(v) < 2:
        raise L.ZkeError("bad G1 point")
    if len(v) >= 3 and _dec(v[2]) == 0:
        return bytes(64)
    return _fq_bytes(v[0]) + _fq_bytes(v[1])


def _g2_bytes(v) -> bytes:
    if not isinstance(v, list) or len(v) < 2 or any(not isinstance(c, list) or len(c) != 2 for c in v[:2]):
        raise L.ZkeError("bad G2 point")
    if len(v) >= 3 and isinstance(v[2], list) and len(v[2]) == 2 and _dec(v[2][0]) == 0 and _dec(v[2][1]) == 0:
        return bytes(128)
    return _fq_bytes(v[0][0]) + _fq_bytes(v[0][1]) + _fq_bytes(v[1][0]) + _fq_bytes(v[1][1])


class Verifier:
    """Groth16 verification on GPU `device` for many proofs under one key (zke_verifier_*; snarkjs.groth16.verify,
    /root/reference/packages/helpers/src/chunked-zkey.ts:101, batched).  Opening validates the key and precomputes its
    fixed pairing data on the GPU.  Each call validates every proof, checks all of them with one randomised product of
    pairings, and only if that fails verifies them one by one - the verdicts of the host `verify_batch`."""

    def __init__(self, vkey: dict, device: int = 0):
        self._h = None
        err = ctypes.create_string_buffer(L.ERRCAP)
        h = L.zke_verifier_open(json.dumps(vkey).encode(), device, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        self._h, self.device, self.n_public = h, device, len(vkey["IC"]) - 1

    def close(self):
        if getattr(self, "_h", None):
            L.zke_verifier_close(self._h)
            self._h = None

    __del__ = close

    def verify_batch_raw(self, proofs256: bytes, publics: bytes, n: int, rand: bytes | None = None) -> list:
        """n proofs in zke_prove's layout ([n][8][32]) with their public signals ([n][n_public][32]) - the output of
        Context.prove - checked on the GPU.  rand: 16 bytes per proof (default: drawn by the library)."""
        if n < 0 or len(proofs256) < 256 * n or len(publics) < 32 * self.n_public * n:
            raise ValueError("proof or public-signal buffer shorter than n entries")
        if rand is not None and len(rand) != 16 * n:
            raise ValueError("rand must hold 16 bytes per proof")
        if n == 0:
            return []
        ok = ctypes.create_string_buffer(n)
        err = ctypes.create_string_buffer(L.ERRCAP)
        rc = L.zke_verifier_batch(self._h, n, bytes(proofs256), bytes(publics) if publics else None,
                                  bytes(rand) if rand is not None else None, ok, err, L.ERRCAP)
        if rc < 0:
            raise L.ZkeError(err.value.decode())
        return [b == 1 for b in ok.raw[:n]]

    def verify_batch(self, public_signals_list, proofs, rand: bytes | None = None) -> list:
        """Same arguments, errors and verdicts as the module-level verify_batch, on the GPU."""
        import os
        n = len(proofs)
        if len(public_signals_list) != n:
            raise ValueError("one public-signal list per proof")
        if n == 0:
            return []
        rand = os.urandom(16 * n) if rand is None else rand
        if len(rand) != 16 * n:
            raise ValueError("rand must hold 16 bytes per proof")
        pb, sb = bytearray(), bytearray()
        for sig, pr in zip(public_signals_list, proofs):
            prot = pr.get("protocol")
            if prot is not None and prot != "groth16":
                raise L.ZkeError("proof protocol is not groth16")
            missing = [k for k in ("pi_a", "pi_b", "pi_c") if k not in pr]
            if missing:
                raise L.ZkeError(f"missing key '{missing[0]}'")
            a, b, c = _g1_bytes(pr["pi_a"]), _g2_bytes(pr["pi_b"]), _g1_bytes(pr["pi_c"])
            if not isinstance(sig, list):
                raise L.ZkeError("public signals must be an array per proof")
            vals = [_dec(s) for s in sig]
            if len(vals) != self.n_public:
                # the binary layout has n_public slots: send the proof with an off-curve A, which makes it invalid on the
                # GPU exactly as the wrong count does on the host
                a, vals = _OFF_CURVE_A, [0] * self.n_public
            pb += a + b + c
            sb += b"".join(x.to_bytes(32, "little") for x in vals)
        return self.verify_batch_raw(bytes(pb), bytes(sb), n, bytes(rand))


def verify(vkey: dict, public_signals, proof: dict) -> bool:
    """snarkjs.groth16.verify(vkey, publicSignals, proof) (/root/reference/packages/helpers/src/chunked-zkey.ts:101)."""
    err = ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_verify_json(json.dumps(vkey).encode(), json.dumps([str(s) for s in public_signals]).encode(),
                           json.dumps(proof).encode(), err, L.ERRCAP)
    if rc < 0:
        raise L.ZkeError(err.value.decode())
    return rc == 1
