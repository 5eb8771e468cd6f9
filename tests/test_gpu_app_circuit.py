"""Email app circuits on the GPU (Circuit.from_spec): the witness kernel against the CPU oracle, bit for bit, for the
multi-regex app of tests/test_app_circuit.py and for bare regexes of 65..255 DFA states, which the kernel seeds in its wide
mode (witness.cu: regex_coop, a 256-bit live set) - the oracle walks only the instance's own ops, so these comparisons are
what checks that mode.  Then Groth16 proofs of the app: equal to the oracle's at fixed (r, s), accepted by every verifier,
and fullProve's public signals decode to the revealed strings."""
import ctypes
import json

import pytest

import zkemail_b200 as z
import zkutil
from zkutil import oracle_witness
from test_app_circuit import EXPECTED, RECIPIENT, WIDE_CASES, app_spec, signed_app_email, wide_regex_messages

pytestmark = pytest.mark.gpu

_CACHE = {}


def _app(style):
    if style not in _CACHE:
        spec = app_spec(style)
        c = z.Circuit.from_spec(spec)
        inputs = [z.generate_app_inputs(signed_app_email(i, f"Order #{40213 + 7 * (i - 3)} shipped to {name}"), spec, {"recipient": RECIPIENT})
                  for i, name in ((3, "Alice"), (4, "Bob"))]
        _CACHE[style] = (spec, c, inputs, [oracle_witness(c, x).raw() for x in inputs])
    return _CACHE[style]


def _run(c, inputs, refs, order):
    ctx = z.Context(c, None, device=0, max_batch=len(order))
    packed = b"".join(c.pack_inputs(inputs[e]) for e in order)
    wt, status = ctx.witness(packed, len(order))
    m = 32 * c.info.n_vars
    assert status == [-1] * len(order)
    for k, e in enumerate(order):
        assert wt[k * m:(k + 1) * m] == refs[e], f"email {k} (input {e}) differs from the oracle"


@pytest.mark.parametrize("width", ["default", "1", "8"])
@pytest.mark.parametrize("style", [0, 1], ids=["zkregex", "compact"])
def test_app_witness_matches_oracle(style, width, monkeypatch):
    if width == "default":
        monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    _, c, inputs, refs = _app(style)
    _run(c, inputs, refs, [0, 1, 1, 0])


@pytest.mark.parametrize("width", ["default", "1", "8"])
@pytest.mark.parametrize("case", list(WIDE_CASES))
def test_wide_regex_witness_matches_oracle(case, width, monkeypatch):
    """Messages with a state >= 64 live at every chunk boundary of the wide run and UTF-8 / other bytes >= 0x80 in between
    (tests/test_app_circuit.py: wide_regex_messages; test_wide_seed_record_matches_oracle checks they do that)."""
    monkeypatch.setenv("ZKE_REGEX_STYLE", "0")
    if width == "default":
        monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    c = z.Circuit.from_regex(WIDE_CASES[case][0], 1024)
    inputs = [{"msg": m} for m in wide_regex_messages(case)]
    refs = [oracle_witness(c, x).raw() for x in inputs]
    _run(c, inputs, refs, [0, 1, 2, 3])


def test_app_proof(monkeypatch):
    """Compact shape (2^21 domain: the oracle's prover stays within the suite's time budget)."""
    from oracle import bn254
    monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    spec, c, inputs, refs = _app(1)
    zk = z.Zkey(c, seed=13)
    ctx = z.Context(c, zk, device=0, max_batch=1)
    wt, status = ctx.witness(c.pack_inputs(inputs[0]), 1)
    assert status == [-1] and wt == refs[0]
    r, s = 424242, 171717
    proofs, publics, _ = ctx.prove(1, r.to_bytes(32, "little") + s.to_bytes(32, "little"))
    assert proofs == zkutil.oracle_prove(c, zkutil.product_sections(zk), wt, r, s)
    proof, pubs = z.proof_to_json(proofs, publics, c.info.n_public)
    vk = zk.vkey()
    assert bn254.groth16_verify(vk, pubs, proof) and z.verify(vk, pubs, proof)
    assert z.Verifier(vk, device=0).verify_batch([pubs], [proof]) == [True]
    out = z.decode_app_outputs(spec, pubs)
    assert {k: out[k] for k in EXPECTED} == EXPECTED

    # fullProve from the input JSON: the public signals carry the revealed strings of the second email
    pl, sl = ctypes.c_size_t(1 << 16), ctypes.c_size_t(1 << 16)
    pj, sj = ctypes.create_string_buffer(pl.value), ctypes.create_string_buffer(sl.value)
    err = ctypes.create_string_buffer(z._lib.ERRCAP)
    rc = z._lib.zke_fullprove_json(ctx._h, c.handle, json.dumps(inputs[1]).encode(), pj, ctypes.byref(pl), sj, ctypes.byref(sl),
                                   err, z._lib.ERRCAP)
    assert rc == 0, err.value
    pubs2, proof2 = json.loads(sj.value), json.loads(pj.value)
    out2 = z.decode_app_outputs(spec, pubs2)
    assert (out2["order0"], out2["order1"], out2["fromAddress"]) == ("40220", "Bob", "sender0004@gmail.com")
    assert z.verify(vk, pubs2, proof2)
    tampered = list(pubs2)
    tampered[-2] = str(int(tampered[-2]) + 1)                # the recipient is bound to the proof
    assert not z.verify(vk, tampered, proof2)
