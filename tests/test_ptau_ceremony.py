"""Phase-1 `.ptau` verbs that need no GPU: ptau_new against the Python writer, and the refusals that come before any device
work (the reader's optional Lagrange sections, an already prepared file, bad contribution secrets, argument errors)."""
import ctypes

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from ptau_writer import R, write_ptau

UNPREPARED = {12: None, 13: None, 14: None, 15: None}


@pytest.mark.parametrize("power", [1, 4, 11])
def test_ptau_new_equals_the_python_writer(power):
    assert bytes(z.ptau_new(power)) == write_ptau(power, overrides=UNPREPARED)[0]


def test_ptau_new_refuses_powers_out_of_range():
    for p in (0, 29):
        with pytest.raises(L.ZkeError, match=r"\[1, 28\]"):
            z.ptau_new(p)


def test_reader_needs_all_or_none_of_the_lagrange_sections():
    for missing, name in ((13, "lTauG2"), (15, "lBetaTauG1")):
        partial = write_ptau(2, overrides={missing: None})[0]
        for verb in (lambda f: z.ptau_contribute(f, (2, 3, 4)), z.ptau_prepare, z.verify_ptau):
            with pytest.raises(L.ZkeError, match=f"section {missing} \\({name}\\) is missing"):
                verb(partial)
    # the strict reader of from_ptau / ptau_info is unchanged: an unprepared file is refused as before
    with pytest.raises(L.ZkeError, match=r"section 12 \(lTauG1\) is missing"):
        z.ptau_info(z.ptau_new(3))
    with pytest.raises(L.ZkeError, match="already prepared"):
        z.ptau_prepare(write_ptau(2)[0])


def test_contribution_secrets_are_refused_by_name():
    new = z.ptau_new(2)
    for bad, what in ((0, "zero"), (1, "one"), (R, "not below the group order r")):
        for i, name in enumerate(("tau", "alpha", "beta")):
            s = [5, 6, 7]
            s[i] = bad
            with pytest.raises(L.ZkeError, match=f"secret {name} is {what}"):
                z.ptau_contribute(new, tuple(s))


def test_prev_and_receipt_go_together():
    new = bytes(z.ptau_new(1))
    err = ctypes.create_string_buffer(L.ERRCAP)
    assert L.zke_ptau_verify(new, len(new), new, len(new), None, None, 0, err, L.ERRCAP) < 0
    assert "give both or neither" in err.value.decode()
    assert L.zke_ptau_verify(new, len(new), None, 0, bytes(384), None, 0, err, L.ERRCAP) < 0
    with pytest.raises(ValueError):
        z.verify_ptau(new, prev=new)
