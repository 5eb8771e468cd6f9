"""Hashed and committed reveals on the GPU: the witness kernel's native Poseidon op (witness.cu: poseidon_coop) against
the CPU oracle, bit for bit - the oracle walks the gadgets' own ops, so these comparisons are what checks the op - with
the op on and off, in both regex shapes, at cluster widths default, 1 and 8.  The inputs hold a maximum-length reveal
(the 5-digit order id), a reveal of 600 bytes (two chained chunk hashes) and a salt of r - 1.  Then the app's proof at
fixed (r, s) against the oracle's, under every verifier, and fullProve's public signals against expected_app_output."""
import ctypes
import json

import pytest

import zkemail_b200 as z
import zkutil
from zkutil import oracle_witness
from test_app_commit import LONG_NOTE, SALT, commit_spec, sender_of, signed_commit_email

pytestmark = pytest.mark.gpu

R = z.FR_MODULUS
_CACHE = {}
# (email index, order id, note, salt)
CASES = [(3, "40213", LONG_NOTE, SALT), (4, "7", "short note", R - 1)]


def _app(style):
    if style not in _CACHE:
        spec = commit_spec(style)
        c = z.Circuit.from_spec(spec)
        inputs = [z.generate_app_inputs(signed_commit_email(i, order, note), spec, {"senderSalt": salt, "recipient": 5 + i})
                  for i, order, note, salt in CASES]
        _CACHE[style] = (spec, c, inputs, [oracle_witness(c, x).raw() for x in inputs])
    return _CACHE[style]


@pytest.mark.parametrize("native", ["1", "0"], ids=["native", "gadget"])
@pytest.mark.parametrize("width", ["default", "1", "8"])
@pytest.mark.parametrize("style", [0, 1], ids=["zkregex", "compact"])
def test_commit_witness_matches_oracle(style, width, native, monkeypatch):
    if width == "default":
        monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("ZKE_WITNESS_CLUSTER", width)
    monkeypatch.setenv("ZKE_NATIVE_POSEIDON", native)
    _, c, inputs, refs = _app(style)
    order = [0, 1, 1, 0]
    ctx = z.Context(c, None, device=0, max_batch=len(order))
    wt, status = ctx.witness(b"".join(c.pack_inputs(inputs[e]) for e in order), len(order))
    m = 32 * c.info.n_vars
    assert status == [-1] * len(order)
    for k, e in enumerate(order):
        assert wt[k * m:(k + 1) * m] == refs[e], f"email {k} (input {e}) differs from the oracle"


def test_commit_proof(monkeypatch):
    """Compact shape (2^21 domain: the oracle's prover stays within the suite's time budget)."""
    from oracle import bn254
    monkeypatch.delenv("ZKE_WITNESS_CLUSTER", raising=False)
    monkeypatch.delenv("ZKE_NATIVE_POSEIDON", raising=False)
    spec, c, inputs, refs = _app(1)
    zk = z.Zkey(c, seed=19)
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

    # fullProve of the second email (salt r - 1): the outputs are what the host computes from the plain values
    pl, sl = ctypes.c_size_t(1 << 16), ctypes.c_size_t(1 << 16)
    pj, sj = ctypes.create_string_buffer(pl.value), ctypes.create_string_buffer(sl.value)
    err = ctypes.create_string_buffer(z._lib.ERRCAP)
    rc = z._lib.zke_fullprove_json(ctx._h, c.handle, json.dumps(inputs[1]).encode(), pj, ctypes.byref(pl), sj, ctypes.byref(sl),
                                   err, z._lib.ERRCAP)
    assert rc == 0, err.value
    pubs2, proof2 = json.loads(sj.value), json.loads(pj.value)
    out = z.decode_app_outputs(spec, pubs2)
    i, order, note, salt = CASES[1]
    assert out["sender"] == z.expected_app_output(spec, "sender", sender_of(i), salt)
    assert out["order"] == z.expected_app_output(spec, "order", order)
    assert out["note"] == z.expected_app_output(spec, "note", note)
    assert out["recipient"] == 5 + i
    assert z.verify(vk, pubs2, proof2)
    tampered = list(pubs2)
    tampered[3] = str(z.expected_app_output(spec, "sender", sender_of(i), SALT))     # another salt's commitment
    assert not z.verify(vk, tampered, proof2)
