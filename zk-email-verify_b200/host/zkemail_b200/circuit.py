"""Circuit handle: the role `wasm_tester(circuitFile)` / the `.r1cs + .wasm` pair play in the reference
(/root/reference/packages/circuits/tests/email-verifier.test.ts:21-31)."""
from __future__ import annotations
import ctypes
from . import _lib as L
from ._mapped import mapped_buffer

FR_MODULUS = 21888242871839275222246405745257275088548364400416034343698204186575808495617
R1CS_NO_PROGRAM = ("this circuit was read from an .r1cs: it has no witness program "
                   "(load witnesses with zke_load_witness / zke_wtns_prove)")


class Circuit:
    def __init__(self, template: str, params=(), _handle=None):
        if _handle is None:
            arr = (L.c_i64 * len(params))(*[int(p) for p in params])
            err = ctypes.create_string_buffer(L.ERRCAP)
            _handle = L.zke_circuit_build(template.encode(), arr, len(params), err, L.ERRCAP)
            if not _handle:
                raise L.ZkeError(err.value.decode())
        self._h = _handle
        self.template, self.params = template, tuple(params)
        info = L.CircuitInfo()
        L.zke_circuit_get_info(self._h, ctypes.byref(info))
        self.info = info
        self.groups = {}
        name = ctypes.create_string_buffer(256)
        first, count, kind = L.c_u32(), L.c_u32(), L.c_int()
        for i in range(info.n_groups):
            L.zke_circuit_group(self._h, i, name, 256, ctypes.byref(first), ctypes.byref(count), ctypes.byref(kind))
            self.groups[name.value.decode()] = (first.value, count.value, kind.value)

    @classmethod
    def from_regex(cls, parts, msg_len: int):
        """zk-regex circuit of a decomposed regex: parts = [(regex fragment, is_public), ...]; signals msg[msg_len] ->
        out, reveal0[msg_len] (the generator behind BodyHashRegex, email-verifier.circom:5,126)."""
        arr = (L.c_char_p * len(parts))(*[p.encode() for p, _ in parts])
        pub = bytes(1 if q else 0 for _, q in parts)
        err = ctypes.create_string_buffer(L.ERRCAP)
        h = L.zke_circuit_build_regex(arr, pub, len(parts), msg_len, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return cls("Regex", (msg_len,), _handle=h)

    @classmethod
    def from_spec(cls, spec):
        """An email app circuit from its spec (a dict or its JSON text; layout in app.py and at zke_circuit_build_app):
        EmailVerifier with its flags, then the app's regexes with their revealed parts, external public inputs and an
        optional email nullifier.  Witnesses and proofs run on the GPU like any template circuit."""
        import json
        text = spec if isinstance(spec, str) else json.dumps(spec)
        err = ctypes.create_string_buffer(L.ERRCAP)
        h = L.zke_circuit_build_app(text.encode(), err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        c = cls("EmailApp", (), _handle=h)
        c.spec = json.loads(text)
        return c

    @classmethod
    def from_r1cs(cls, src):
        """circom's constraint system: an iden3 `.r1cs` (bytes, a buffer or a path, which is memory-mapped), as `circom
        --r1cs` writes it for `snarkjs groth16 setup`.  The circuit has no witness program: its witnesses come from circom's
        witness calculator (Context.load_witness / wtns_prove), and key setup, contributions and proving work as usual."""
        err = ctypes.create_string_buffer(L.ERRCAP)
        with mapped_buffer(src) as (ptr, n):
            h = L.zke_circuit_from_r1cs(ptr, n, err, L.ERRCAP)
        if not h:
            raise L.ZkeError(err.value.decode())
        return cls("r1cs", (), _handle=h)

    def write_r1cs(self) -> bytes:
        """The constraint system as an `.r1cs` image, written natively: the bytes of iden3_binfile.write_r1cs, and for a
        circuit read with from_r1cs its labels and constraints as they were read."""
        n = L.zke_circuit_write_r1cs(self._h, None, 0)
        if n < 0:
            raise L.ZkeError("r1cs export failed")
        buf = ctypes.create_string_buffer(n)
        if L.zke_circuit_write_r1cs(self._h, buf, n) != n:
            raise L.ZkeError("r1cs export failed")
        return buf.raw

    def __del__(self):
        if getattr(self, "_h", None):
            L.zke_circuit_free(self._h)
            self._h = None

    @property
    def handle(self):
        return self._h

    @property
    def n_inputs(self):
        return self.info.n_pub_inputs + self.info.n_prv_inputs

    def pack_inputs(self, inputs: dict) -> bytes:
        """snarkjs input JSON ({name: decimal string | number | list}) -> [n_inputs][32] little-endian bytes,
        in witness order.  Mirrors the checks of circom_runtime's witness calculator: every declared input
        must be present with the right number of values ("Not all inputs have been set" / "Too many values")."""
        if self.template == "r1cs":
            raise L.ZkeError(R1CS_NO_PROGRAM)
        base = 1 + self.info.n_outputs
        buf = bytearray(32 * self.n_inputs)
        seen = set()
        for name, val in inputs.items():
            if name not in self.groups or self.groups[name][2] == 0:
                raise L.ZkeError(f"Signal not found: {name}")
            first, count, _ = self.groups[name]
            flat = _flatten(val)
            if len(flat) != count:
                raise L.ZkeError(f"{'Too many' if len(flat) > count else 'Not enough'} values for input signal {name}")
            for i, v in enumerate(flat):
                x = int(v) % FR_MODULUS
                off = 32 * (first - base + i)
                buf[off:off + 32] = x.to_bytes(32, "little")
            seen.add(name)
        for name, (_, _, kind) in self.groups.items():
            if kind != 0 and name not in seen:
                raise L.ZkeError(f"Not all inputs have been set. Missing: {name}")
        return bytes(buf)

    def array(self, which: int, ctype):
        n = L.c_size_t()
        p = L.zke_circuit_array(self._h, which, ctypes.byref(n))
        return p, n.value

    def program_stats(self, native_sha=True, native_regex=True, coop_fpmul=True, cluster=1, native_poseidon=True) -> dict:
        """What the engine's lowering of the witness program (csrc/witness_program.cpp) builds for these options, computed
        on the host: the fields of zke_program_stats plus `level_ops`, the records per level that are not cooperative ops."""
        st, err = L.ProgramStats(), ctypes.create_string_buffer(L.ERRCAP)
        flags = ((L.LOWER_NATIVE_SHA if native_sha else 0) | (L.LOWER_NATIVE_REGEX if native_regex else 0) |
                 (L.LOWER_COOP_FPMUL if coop_fpmul else 0) | (L.LOWER_NATIVE_POSEIDON if native_poseidon else 0))
        cap = max(1, self.info.n_levels)
        while True:                # the first min(n_levels, cap) levels are written: once more if the program got deeper
            level_ops = (L.c_u32 * cap)()
            if L.zke_circuit_program_stats_ex(self._h, flags, cluster, ctypes.byref(st), level_ops, cap, err, L.ERRCAP) != 0:
                raise L.ZkeError(err.value.decode())
            if st.n_levels <= cap:
                break
            cap = st.n_levels
        out = {name: getattr(st, name) for name, _ in st._fields_}
        out["level_ops"] = list(level_ops[:st.n_levels])
        return out

    def scope_name(self, idx: int) -> str:
        s = L.zke_circuit_scope_name(self._h, idx)
        return s.decode() if s else "?"


def r1cs_info(src) -> dict:
    """`snarkjs r1cs info`: the fields it prints for an `.r1cs` (bytes, a buffer or a path).  The whole file is read and
    checked as Circuit.from_r1cs does; nLabels comes from its header."""
    import struct
    c = Circuit.from_r1cs(src)
    with mapped_buffer(src) as (ptr, n):
        view = (ctypes.c_char * n).from_address(ptr) if isinstance(ptr, int) else ptr
        n_sec, pos, labels = struct.unpack_from("<I", view, 8)[0], 12, None
        for _ in range(n_sec):
            typ, size = struct.unpack_from("<IQ", view, pos)
            if typ == 1:
                labels = struct.unpack_from("<Q", view, pos + 12 + 4 + 32 + 16)[0]
                break
            pos += 12 + size
        del view
    i = c.info
    return {"curve": "bn128", "wires": i.n_vars, "constraints": i.n_constraints, "private_inputs": i.n_prv_inputs,
            "public_inputs": i.n_pub_inputs, "outputs": i.n_outputs, "labels": labels}


def _flatten(v):
    if isinstance(v, (list, tuple)):
        out = []
        for x in v:
            out.extend(_flatten(x))
        return out
    return [v]
