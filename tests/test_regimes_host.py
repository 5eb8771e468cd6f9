"""Host side of the prover-regime tests (tests/test_gpu_regimes.py): the size- and content-controlled R1CS generator lands
in the domain it is asked for, its witness satisfies the rows, and every class of adversarial multi-exponentiation input
is present; the CPU oracle's own prover, on the adversarial instance, gives a proof the pairing check accepts; and the
witness program is a different stream at each cluster width the GPU tests compare.  No GPU needed."""
import ctypes
import time

import numpy as np
import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from oracle import bn254
from r1cs_gen import (A_ONLY, F_SHARED, HEAVY_BUCKET, N_OUT, N_PRV, N_PUB, N_PUBLIC, OPPOSITE_SCALARS, SMALL, SPECIAL,
                      UNUSED, generate, value, window_ones)
from test_r1cs_reader import R, _arr, circuit_rows
from zkutil import oracle_prove, oracle_setup, proof_json_from_bytes, ref, ref_view, vkey_from_sections


def _check(c, witness):
    return ref.zkref_check_r1cs(ctypes.byref(ref_view(c)), witness)


def _occurrences(c, n_wires):
    """Per wire: how many terms name it in A, B and C."""
    return [np.bincount(_arr(c, which, np.uint32), minlength=n_wires) for which in (L.ARR_A_VAR, L.ARR_B_VAR, L.ARR_C_VAR)]


@pytest.mark.parametrize("log_n,heavy", [(8, False), (10, True), (13, True), (17, True), (20, True)])
def test_generator_domain_witness_and_classes(log_n, heavy):
    t0 = time.perf_counter()
    g = generate(log_n, heavy=heavy)
    assert time.perf_counter() - t0 < 30
    c = z.Circuit.from_r1cs(g["blob"])
    i = c.info
    assert i.domain_log2 == log_n and i.n_constraints == g["n_rows"] and i.n_vars == g["n_wires"]
    assert (i.n_outputs, i.n_pub_inputs, i.n_prv_inputs, i.n_public) == (N_OUT, N_PUB, N_PRV, N_PUBLIC)
    assert _check(c, g["witness"]) == -1
    # a wrong product is caught at its own row
    x, y, zz = (int(w) for w in g["classes"]["quadratic"][3])
    assert (value(g, x) * value(g, y) - value(g, zz)) % R == 0
    bad = bytearray(g["witness"])
    bad[32 * zz:32 * zz + 32] = ((value(g, zz) + 1) % R).to_bytes(32, "little")
    assert _check(c, bytes(bad)) == g["quad_rows"][3]

    cl, vals = g["classes"], g["values"]
    as_int = lambda ws: [value(g, int(w)) for w in ws]
    assert as_int(cl["identical_one"]) == [1] * 16 and as_int(cl["identical_full"]) == [F_SHARED] * 16
    small = cl["identical_small"]
    assert (vals[small, 0] == SMALL).all() and (vals[small, 1:] == 0).all()
    assert (len(small) > HEAVY_BUCKET) == heavy
    p, q = cl["opposite_p"], cl["opposite_q"]
    assert as_int(p) == as_int(q) and as_int(p)[:len(OPPOSITE_SCALARS)] == OPPOSITE_SCALARS
    assert as_int(cl["a_only"]) == A_ONLY and as_int(cl["unused"]) == UNUSED and as_int(cl["special"]) == SPECIAL
    for v in (0, 1, R - 1, (R - 1) // 2, (R + 1) // 2, (1 << 253) - 1, window_ones(8), window_ones(12), window_ones(17),
              window_ones(20)):
        assert v in SPECIAL
    bits = vals[cl["bit"]]
    assert set(bits[:, 0].tolist()) == {0, 1} and not bits[:, 1:].any()
    sm = vals[cl["small"]]
    assert sm[:, 0].min() >= 2 and sm[:, 0].max() < 256 and not sm[:, 1:].any()
    assert len(cl["bit"]) > 2 * (len(cl["small"]) + len(cl["full_width"]))          # mostly bits, as in EmailVerifier
    assert (vals[cl["full_width"], 3] >> np.uint64(58)).any()                         # full width: values above 2^250

    # where the wires occur: equal columns for the shared rows, none for the unused wires, A only for the A-only wires
    occ_a, occ_b, occ_c = _occurrences(c, g["n_wires"])
    ident = np.concatenate([cl["identical_one"], cl["identical_full"], small])
    for occ, k in ((occ_a, 1), (occ_b, 1), (occ_c, 2)):            # (sum u) * 1 = sum u, 1 * (sum u) = sum u
        assert (occ[ident] == k).all() and (occ[p] == k).all() and (occ[q] == k).all()
        assert (occ[cl["unused"]] == 0).all()
    assert (occ_a[cl["a_only"]] == 1).all() and (occ_b[cl["a_only"]] == 0).all() and (occ_c[cl["a_only"]] == 0).all()
    qd = cl["quadratic"]
    assert (occ_a[qd[:, 0]] == 1).all() and (occ_b[qd[:, 1]] == 1).all() and (occ_c[qd[:, 2]] == 1).all()
    assert (occ_b[qd[:, 0]] == 0).all() and (occ_a[qd[:, 2]] == 0).all()


def test_points_of_the_shared_and_opposite_rows():
    """On a small instance, row by row: every shared-row wire has the same (row, coefficient) column in A, B and C, and
    each q of an opposite pair has its p's column negated - so their key points are equal, or opposite."""
    g = generate(8, heavy=False)
    rows = circuit_rows(z.Circuit.from_r1cs(g["blob"]))
    cols = {}
    for r, row in enumerate(rows):
        for m, lc in enumerate(row):
            for w, k in lc:
                cols.setdefault(w, []).append((m, r, k))
    cl = g["classes"]
    ident = np.concatenate([cl["identical_one"], cl["identical_full"], cl["identical_small"]])
    assert len({tuple(cols[int(w)]) for w in ident}) == 1
    for p, q in zip(cl["opposite_p"], cl["opposite_q"]):
        assert [(m, r, (R - k) % R) for m, r, k in cols[int(p)]] == cols[int(q)]
    assert all(int(w) not in cols for w in cl["unused"])
    assert all({m for m, _, _ in cols[int(w)]} == {0} for w in cl["a_only"])


def test_oracle_proves_the_adversarial_instance():
    """The oracle's prover (the reference the GPU proofs are compared with) on identical and opposite points, zero, one,
    r - 1, (r -+ 1) / 2 and carry-through-every-window scalars, points at infinity: the pairing check accepts its proof."""
    g = generate(8, heavy=False)
    c = z.Circuit.from_r1cs(g["blob"])
    sec = oracle_setup(c, (0x1234567890ABCDEF1234567, 0x2222222222222222222333, 0x3333333333444, 0x44444444444445555,
                           0x5555555566666))
    vk = vkey_from_sections(sec, N_PUBLIC)
    pubs = [str(value(g, 1 + i)) for i in range(N_PUBLIC)]
    proof = oracle_prove(c, sec, g["witness"], 0x1234567890ABCDEF, 0xFEDCBA0987654321, threads=4)
    assert bn254.groth16_verify(vk, pubs, proof_json_from_bytes(proof))
    bad = [pubs[0], str((int(pubs[1]) + 1) % R)]
    assert not bn254.groth16_verify(vk, bad, proof_json_from_bytes(proof))


# ------------------------------------------------------------------------------------------------ witness cluster widths
# the circuits tests/test_gpu_regimes.py runs at each cluster width
CLUSTER_CIRCUITS = [("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1]), ("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1, 1]),
                    ("Sha256Bytes", [128]), ("Sha256Bytes", [192]), ("FpMul", [121, 17]), ("Poseidon", [2])]


@pytest.mark.parametrize("template,params", CLUSTER_CIRCUITS, ids=["email", "email_compact", "sha128", "sha192", "fpmul", "poseidon"])
def test_each_cluster_width_is_its_own_stream(template, params):
    """The lowering pads every level to whole rounds of `cluster` iterations: the four widths give four different streams,
    so the four GPU comparisons per circuit check four different programs."""
    c = z.Circuit(template, params)
    st = {w: c.program_stats(cluster=w) for w in (1, 2, 4, 8)}
    for w, s in st.items():
        assert s["cluster"] == w and s["n_iters"] % w == 0
    assert len({s["digest"] for s in st.values()}) == 4
    if (template, params) == ("Sha256Bytes", [128]):
        assert [st[w]["n_iters"] for w in (1, 2, 4, 8)] == [12, 20, 36, 72]
    if template == "Poseidon":
        assert [st[w]["n_iters"] for w in (1, 2, 4, 8)] == [261, 522, 1044, 2088]
