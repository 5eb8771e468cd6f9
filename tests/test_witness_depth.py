"""Depth of the witness program the engine runs, as its own lowering builds it (csrc/witness_program.cpp through
zke_circuit_program_stats; scripts/witness_depth.py prints the same figures): the native SHA-256 op and the regex state
seeding must keep collapsing the long dependency chains - a regression in the records the front end emits (circuit.hpp:
ShaBlock, RegexSeed) or in the lowering shows up here as a jump in levels / iterations, long before it costs milliseconds
on the GPU.  The padding to cluster rounds, the FpMul record and the determinism of the stream are checked on the CPU too."""
import os
import sys

import numpy as np
import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import witness_depth


def test_regex_template_collapses_to_a_few_levels():
    for style in (0, 1):
        c = z.Circuit("BodyHashRegex", [128, style])
        plain = witness_depth.analyse(c, True, False)
        seeded = witness_depth.analyse(c, True, True)
        assert plain[0] > 200 and seeded[0] <= 16, (style, plain[0], seeded[0])        # ~2-5 levels per byte -> a handful in total
        assert seeded[2] == plain[2]                                                  # every op is kept
        assert seeded[1] < plain[1]


def test_email_verifier_test_circuit_depth():
    c = z.Circuit("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1])
    generic = witness_depth.analyse(c, False, False)
    sha = witness_depth.analyse(c, True, False)
    both = witness_depth.analyse(c, True, True)
    assert generic[0] > sha[0] > both[0]
    assert both[0] <= 400                       # what is left is the Poseidon round chain of the public-key hash
    assert both[1] <= 1.25 * (-(-both[2] // witness_depth.T))    # within 25 % of the 512-ops-per-iteration floor


@pytest.mark.parametrize("template,params", [("BodyHashRegex", [128]), ("Sha256Bytes", [64])])
def test_levels_are_padded_to_whole_cluster_rounds(template, params):
    c = z.Circuit(template, params)
    one = c.program_stats(cluster=1)
    assert sum(one["level_ops"]) == one["n_ops_kept"] and len(one["level_ops"]) == one["n_levels"]
    for cluster in (1, 2, 4, 8):
        st = c.program_stats(cluster=cluster)
        assert st["cluster"] == cluster and st["n_iters"] % cluster == 0
        assert (st["n_levels"], st["n_ops_kept"], st["level_ops"]) == (one["n_levels"], one["n_ops_kept"], one["level_ops"])
        assert st["n_iters"] >= one["n_iters"]
    with pytest.raises(L.ZkeError, match="cluster must be"):
        c.program_stats(cluster=3)


def test_sequential_fpmul_is_a_regular_record():
    c = z.Circuit("FpMul", [121, 17])
    p, n = c.array(L.ARR_OPS, None)
    ops = np.ctypeslib.as_array((L.c_u32 * (5 * n)).from_address(p)).reshape(n, 5)
    n_fpmul = int((ops[:, 0] == 4).sum())                      # OP_FPMUL
    coop, seq = c.program_stats(coop_fpmul=True), c.program_stats(coop_fpmul=False)
    assert n_fpmul >= 1 and coop["n_coop_ops"] == n_fpmul and seq["n_coop_ops"] == 0
    assert seq["n_levels"] == coop["n_levels"]
    assert seq["n_ops_kept"] == coop["n_ops_kept"] + n_fpmul


def test_lowering_is_deterministic():
    c = z.Circuit("BodyHashRegex", [128])
    a, b = c.program_stats(cluster=4), c.program_stats(cluster=4)
    assert a == b and a["digest"] != 0
    assert c.program_stats(cluster=1)["digest"] != a["digest"]      # the digest covers the padding
    assert c.program_stats(native_regex=False, cluster=4)["digest"] != a["digest"]


def test_r1cs_circuit_has_no_program():
    c = z.Circuit.from_r1cs(z.Circuit("Multiplier").write_r1cs())
    with pytest.raises(L.ZkeError, match="no witness program"):
        c.program_stats()
