"""circom's `.r1cs` read natively (Circuit.from_r1cs) and written natively (Circuit.write_r1cs): byte identity with the
Python writer, the rows as read against an independent list-based parser, a circom-shaped file with the features the
engine's own builder never emits, and every refusal.  Host only: no GPU needed."""
import ctypes
import random
import struct

import numpy as np
import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkemail_b200 import iden3_binfile
from zkemail_b200.circuit import R1CS_NO_PROGRAM
from zkutil import ref, ref_view

R = z.FR_MODULUS
BLS12_381_R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
FQ = 21888242871839275222246405745257275088696311157297823662689037894645226208583


# ------------------------------------------------------------------------------------------------ independent parser
def parse_r1cs(blob: bytes) -> dict:
    """Every term as written, in file order (duplicate wires and zero coefficients kept); sections in any order."""
    assert blob[:4] == b"r1cs"
    version, n_sec = struct.unpack_from("<II", blob, 4)
    pos, sec = 12, {}
    for _ in range(n_sec):
        typ, size = struct.unpack_from("<IQ", blob, pos)
        sec[typ] = blob[pos + 12:pos + 12 + size]
        pos += 12 + size
    assert pos == len(blob)
    h = sec[1]
    n8 = struct.unpack_from("<I", h, 0)[0]
    prime = int.from_bytes(h[4:4 + n8], "little")
    n_wires, n_out, n_pub, n_prv, n_labels, n_cons = struct.unpack_from("<IIIIQI", h, 4 + n8)
    body, p, cons = sec[2], 0, []
    for _ in range(n_cons):
        row = []
        for _m in range(3):
            k = struct.unpack_from("<I", body, p)[0]
            p += 4
            lc = []
            for _t in range(k):
                lc.append((struct.unpack_from("<I", body, p)[0], int.from_bytes(body[p + 4:p + 4 + n8], "little")))
                p += 4 + n8
            row.append(lc)
        cons.append(tuple(row))
    assert p == len(body)
    labels = list(struct.unpack_from(f"<{n_wires}Q", sec[3])) if 3 in sec else None
    return {"version": version, "prime": prime, "n_wires": n_wires, "n_out": n_out, "n_pub": n_pub, "n_prv": n_prv,
            "n_labels": n_labels, "constraints": cons, "labels": labels}


def circuit_rows(c: z.Circuit) -> list:
    """The circuit's rows as (A, B, C) lists of (wire, coefficient value), from its exported arrays."""
    coefs = [int.from_bytes(b, "little") for b in iden3_binfile._coefs(c)]
    mats = []
    for p, v, k in ((L.ARR_A_PTR, L.ARR_A_VAR, L.ARR_A_COEF), (L.ARR_B_PTR, L.ARR_B_VAR, L.ARR_B_COEF),
                    (L.ARR_C_PTR, L.ARR_C_VAR, L.ARR_C_COEF)):
        mats.append((list(iden3_binfile._u32_array(c, p)), list(iden3_binfile._u32_array(c, v)), list(iden3_binfile._u32_array(c, k))))
    return [tuple([(var[i], coefs[cf[i]]) for i in range(ptr[row], ptr[row + 1])] for ptr, var, cf in mats)
            for row in range(c.info.n_constraints)]


def _arr(c, which, dtype, width=1):
    p, n = c.array(which, None)
    if not n:
        return np.zeros((0, width) if width > 1 else 0, dtype=dtype)
    raw = ctypes.string_at(p, n * np.dtype(dtype).itemsize * width)
    a = np.frombuffer(raw, dtype=dtype)
    return a.reshape(n, width) if width > 1 else a


def same_rows(c1: z.Circuit, c2: z.Circuit) -> bool:
    """Row-by-row equality by value (coefficient tables may be interned in different orders), vectorised."""
    k1, k2 = _arr(c1, L.ARR_COEFS, np.uint8, 32), _arr(c2, L.ARR_COEFS, np.uint8, 32)
    for p, v, k in ((L.ARR_A_PTR, L.ARR_A_VAR, L.ARR_A_COEF), (L.ARR_B_PTR, L.ARR_B_VAR, L.ARR_B_COEF),
                    (L.ARR_C_PTR, L.ARR_C_VAR, L.ARR_C_COEF)):
        if not np.array_equal(_arr(c1, p, np.uint32), _arr(c2, p, np.uint32)):
            return False
        if not np.array_equal(_arr(c1, v, np.uint32), _arr(c2, v, np.uint32)):
            return False
        if not np.array_equal(k1[_arr(c1, k, np.uint32)], k2[_arr(c2, k, np.uint32)]):
            return False
    return True


INFO_FIELDS = ("n_vars", "n_outputs", "n_pub_inputs", "n_prv_inputs", "n_public", "n_constraints", "domain_log2",
               "nnz_a", "nnz_b", "nnz_c")


# ------------------------------------------------------------------------------------------------ template circuits
TEMPLATES = [("Multiplier", []), ("FpMul", [2, 4]), ("Sha256Bytes", [64]), ("SelectRegexReveal", [34, 8]),
             ("EmailVerifier", [640, 768, 121, 17])]


@pytest.mark.parametrize("tmpl", TEMPLATES, ids=[t[0] for t in TEMPLATES])
def test_template_circuits_round_trip(tmpl):
    c = z.Circuit(*tmpl)
    blob = c.write_r1cs()
    assert blob == iden3_binfile.write_r1cs(c), "native .r1cs writer differs from the Python writer"
    r = z.Circuit.from_r1cs(blob)
    assert r.template == "r1cs" and r.info.n_ops == 0 and r.info.n_levels == 0 and r.info.n_temps == 0
    for f in INFO_FIELDS:
        assert getattr(r.info, f) == getattr(c.info, f), f
    assert same_rows(r, c)
    assert r.write_r1cs() == blob
    if c.info.nnz_a + c.info.nnz_b + c.info.nnz_c < 200_000:
        assert circuit_rows(r) == parse_r1cs(blob)["constraints"]


# ------------------------------------------------------------------------------------------------ circom-shaped R1CS
N_OUT, N_PUB, N_PRV, N_INT = 2, 3, 4, 300


def _le(x):
    return int(x).to_bytes(32, "little")


def header(n_wires, n_constraints, n_labels, n_out=N_OUT, n_pub=N_PUB, n_prv=N_PRV, prime=R, n8=32):
    return struct.pack("<I", n8) + int(prime).to_bytes(n8, "little") + struct.pack("<IIIIQI", n_wires, n_out, n_pub, n_prv,
                                                                                    n_labels, n_constraints)


def body(cons):
    out = bytearray()
    for row in cons:
        for lc in row:
            out += struct.pack("<I", len(lc))
            for wire, coef in lc:
                out += struct.pack("<I", wire) + _le(coef)
    return bytes(out)


def container(sections, magic=b"r1cs", version=1):
    out = bytearray(magic + struct.pack("<II", version, len(sections)))
    for typ, payload in sections:
        out += struct.pack("<IQ", typ, len(payload)) + payload
    return bytes(out)


def synthetic(seed=1, tweak=False):
    """A circom-shaped R1CS and a satisfying witness: wires [1, outputs, public inputs, private inputs, internals]; each
    constraint defines one fresh wire through its C (quadratic rows with random full-width coefficients, every third row
    linear with empty A and B); one LC names a wire twice, one has a zero coefficient, coefficients r - 1 and 2^200 occur;
    some wires appear in no constraint; labels are not the identity and nLabels > nWires.  tweak: one A coefficient changed
    (the same shape, another circuit)."""
    rng = random.Random(seed)
    first_int = 1 + N_OUT + N_PUB + N_PRV
    n_wires = first_int + N_INT
    unused = set(range(first_int + 7, n_wires, 37))
    fresh = [v for v in range(first_int, n_wires) if v not in unused] + [1, 2]
    w = [0] * n_wires
    w[0] = 1
    for v in list(range(1 + N_OUT, first_int)) + sorted(unused):
        w[v] = rng.randrange(R)
    known = [0] + list(range(1 + N_OUT, first_int))

    def coef():
        k = rng.randrange(6)
        return (1, R - 1, 1 << rng.randrange(1, 253), R - (1 << rng.randrange(1, 253)), rng.randrange(2, 100), rng.randrange(R))[k]

    def lc(n):
        return [(rng.choice(known), coef()) for _ in range(n)]

    def val(terms):
        return sum(c * w[v] for v, c in terms) % R

    cons = []
    for i, f in enumerate(fresh):
        linear = i % 3 == 2
        a, b = ([], []) if linear else (lc(rng.randint(1, 4)), lc(rng.randint(1, 3)))
        cc = lc(rng.randint(0, 3))
        if i == 3:
            x = rng.choice(known)
            a = [(x, 3), (known[1], 7), (x, 5)]          # the same wire twice in one LC
        if i == 4:
            b = b + [(rng.choice(known), 0)]             # a zero coefficient
        if i == 6:
            a = a + [(rng.choice(known), 1 << 200)]
            cc = cc + [(rng.choice(known), R - 1)]
        if tweak and i == 0:
            a = [(a[0][0], (a[0][1] + 1) % R)] + a[1:]
        cf = rng.randrange(1, R)
        pos = rng.randint(0, len(cc))
        row_c = cc[:pos] + [(f, cf)] + cc[pos:]
        w[f] = (val(a) * val(b) - val(cc)) * pow(cf, -1, R) % R
        known.append(f)
        cons.append((a, b, row_c))
    labels = [0] + [3 * i + 1 for i in range(1, n_wires)]
    n_labels = 3 * n_wires + 7
    return {"cons": cons, "witness": w, "n_wires": n_wires, "labels": labels, "n_labels": n_labels, "fresh": fresh}


def tampered(s, row):
    """The witness with the wire that constraint `row` defines changed: `row` is the first constraint it violates."""
    w = list(s["witness"])
    f = s["fresh"][row]
    w[f] = (w[f] + 1) % R
    return w


def synthetic_file(s, order=(2, 1, 3)):
    parts = {1: header(s["n_wires"], len(s["cons"]), s["n_labels"]), 2: body(s["cons"]),
             3: b"".join(struct.pack("<Q", x) for x in s["labels"])}
    return container([(t, parts[t]) for t in order])


def witness_bytes(w):
    return b"".join(_le(x) for x in w)


@pytest.fixture(scope="module")
def syn():
    s = synthetic()
    return s, synthetic_file(s)


def test_synthetic_matches_the_list_parser(syn):
    s, blob = syn
    c = z.Circuit.from_r1cs(blob)
    p = parse_r1cs(blob)
    assert p["constraints"] == [tuple(r) for r in s["cons"]]
    assert circuit_rows(c) == p["constraints"]
    i = c.info
    assert (i.n_vars, i.n_outputs, i.n_pub_inputs, i.n_prv_inputs, i.n_constraints) == \
        (s["n_wires"], N_OUT, N_PUB, N_PRV, len(s["cons"]))
    assert i.n_ops == 0 and i.n_temps == 0 and i.n_groups == 0
    # written back in section order 1, 2, 3 with the labels and nLabels it came with
    back = c.write_r1cs()
    assert back == synthetic_file(s, order=(1, 2, 3))
    q = parse_r1cs(back)
    assert q["labels"] == s["labels"] and q["n_labels"] == s["n_labels"]
    # the interned table: 1, r - 1, then the powers of two, then the rest
    coefs = [int.from_bytes(b, "little") for b in iden3_binfile._coefs(c)]
    assert coefs[:2] == [1, R - 1] and len(set(coefs)) == len(coefs)
    pow2 = [v != 0 and (v & (v - 1) == 0 or (R - v) & (R - v - 1) == 0) for v in coefs[2:]]
    assert pow2 == sorted(pow2, reverse=True) and any(pow2) and not all(pow2)


def test_synthetic_witness_against_the_oracle(syn):
    s, blob = syn
    c = z.Circuit.from_r1cs(blob)
    rc = ref_view(c)
    good = witness_bytes(s["witness"])
    assert ref.zkref_check_r1cs(ctypes.byref(rc), good) == -1
    assert ref.zkref_check_r1cs(ctypes.byref(rc), witness_bytes(tampered(s, 40))) == 40


def test_sections_one_and_two_suffice(syn):
    s, _ = syn
    blob = synthetic_file(s, order=(1, 2))
    c = z.Circuit.from_r1cs(blob)
    assert circuit_rows(c) == [tuple(r) for r in s["cons"]]
    assert parse_r1cs(c.write_r1cs())["labels"] == list(range(s["n_wires"]))


def test_from_r1cs_takes_a_path_and_a_buffer(syn, tmp_path):
    _, blob = syn
    path = tmp_path / "syn.r1cs"
    path.write_bytes(blob)
    for src in (str(path), path, bytearray(blob), memoryview(blob)):
        assert z.Circuit.from_r1cs(src).write_r1cs() == z.Circuit.from_r1cs(blob).write_r1cs()


def test_r1cs_info(syn, tmp_path):
    s, blob = syn
    path = tmp_path / "syn.r1cs"
    path.write_bytes(blob)
    want = {"curve": "bn128", "wires": s["n_wires"], "constraints": len(s["cons"]), "private_inputs": N_PRV,
            "public_inputs": N_PUB, "outputs": N_OUT, "labels": s["n_labels"]}
    assert z.r1cs_info(blob) == want
    assert z.r1cs_info(str(path)) == want
    m = z.Circuit("Multiplier")
    assert z.r1cs_info(m.write_r1cs())["labels"] == m.info.n_vars


def test_no_witness_program(syn):
    _, blob = syn
    c = z.Circuit.from_r1cs(blob)
    with pytest.raises(L.ZkeError, match="read from an .r1cs: it has no witness program"):
        c.pack_inputs({})
    out = ctypes.create_string_buffer(32 * max(1, c.n_inputs))
    err = ctypes.create_string_buffer(L.ERRCAP)
    assert L.zke_pack_inputs_json(c.handle, b"{}", out, len(out), err, L.ERRCAP) < 0
    assert err.value.decode() == R1CS_NO_PROGRAM


# ------------------------------------------------------------------------------------------------ refusals
def _small():
    s = synthetic(seed=5)
    s["cons"] = s["cons"][:12]
    return s


def _refusals():
    s = _small()
    n, nc, nl = s["n_wires"], len(s["cons"]), s["n_labels"]
    h, b = header(n, nc, nl), body(s["cons"])
    lab = b"".join(struct.pack("<Q", x) for x in s["labels"])
    ok = container([(1, h), (2, b), (3, lab)])
    cases = {
        "magic": (b"r1cx" + ok[4:], "bad magic"),
        "version": (container([(1, h), (2, b)], version=2), "version 2 is not supported"),
        "no header": (container([(2, b), (3, lab)]), r"section 1 \(header\) is missing"),
        "no constraints": (container([(1, h), (3, lab)]), r"section 2 \(constraints\) is missing"),
        "header twice": (container([(1, h), (2, b), (1, h)]), "section 1 appears twice"),
        "constraints twice": (container([(1, h), (2, b), (2, b)]), "section 2 appears twice"),
        "truncated file": (ok[:len(ok) - len(lab) - 30], r"truncated \.r1cs \(section"),
        "truncated header": (container([(1, h[:40]), (2, b)]), "truncated .r1cs header"),
        "truncated constraints": (container([(1, header(n, nc + 1, nl)), (2, b)]), "section 2 ends inside constraint 12"),
        "trailing bytes": (container([(1, h), (2, b + bytes(5))]), "trailing bytes in .r1cs section 2"),
        "n8": (container([(1, header(n, nc, nl, n8=48, prime=R)), (2, b)]), "48 bytes, expected 32"),
        "bls12-381": (container([(1, header(n, nc, nl, prime=BLS12_381_R)), (2, b)]), "BLS12-381"),
        "other prime": (container([(1, header(n, nc, nl, prime=FQ)), (2, b)]), "not the BN254 scalar field"),
        "too many signals": (container([(1, header(12, nc, nl, n_prv=9)), (2, b)]), "exceeds nWires"),
        "wire": (container([(1, h), (2, body([([(n, 1)], [(0, 1)], [(0, 1)])] + s["cons"][1:]))]),
                 f"constraint 0: wire {n} is out of range"),
        "coefficient": (container([(1, h), (2, body([([(0, R)], [(0, 1)], [(0, 1)])] + s["cons"][1:]))]), "not below r"),
        "labels size": (container([(1, h), (2, b), (3, lab[:-8])]), r"section 3 \(labels\) has"),
        "gate section 4": (container([(1, h), (2, b), (4, bytes(8))]), r"custom gates \(PLONK\) are not supported"),
        "gate section 5": (container([(1, h), (2, b), (5, bytes(8))]), r"custom gates \(PLONK\) are not supported"),
        "domain": (container([(1, header(n, 1 << 28, nl)), (2, b)]), r"exceeds the largest domain, 2\^28"),
    }
    return ok, cases


def test_refusals():
    ok, cases = _refusals()
    z.Circuit.from_r1cs(ok)
    for name, (blob, msg) in cases.items():
        with pytest.raises(L.ZkeError, match=msg):
            z.Circuit.from_r1cs(blob)
            pytest.fail(f"{name}: accepted")
