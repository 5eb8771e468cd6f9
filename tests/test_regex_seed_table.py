"""The state-seeding record of the zk-regex circuits (circuit.hpp: RegexSeed, ZKE_ARR_REGEX_SEEDS): the engine lets ONE
automaton run per regex instance write every state signal, so that the per-position gadgets of all positions evaluate side
by side instead of as a chain as long as the message (witness.cu: regex_coop, witness_program.cpp).  Checked here on the CPU:
the oracle walks the ordinary witness program, and every recorded signal must hold bit `state` of the live-state set an
independent Python run of the recorded transition table reaches at the recorded position - the values the device op writes.
Role in the reference: the generated zk-regex templates (email-verifier.circom:5,126; un-vendored zk-regex-circom)."""
import ctypes
import random

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkutil import oracle_witness


def _seeds(circuit):
    n = L.c_size_t()
    p = L.zke_circuit_array(circuit.handle, L.ARR_REGEX_SEEDS, ctypes.byref(n))
    flat = list((ctypes.c_uint32 * n.value).from_address(p)) if n.value else [0]
    out, pos = [], 1
    for _ in range(flat[0]):
        nd, nb, ns, lo, hi = flat[pos:pos + 5]; pos += 5
        mode, ns = ns >> 31, ns & 0x7fffffff
        bytes_ = flat[pos:pos + nb]; pos += nb
        unpack = lambda words: [(wd >> (8 * k)) & 0xff for wd in words for k in range(4)]
        table = unpack(flat[pos:pos + 64 * ns]); pos += 64 * ns
        group = None
        if mode == 1:
            group = unpack(flat[pos:pos + 64 * ns]); pos += 64 * ns
        desc = flat[pos:pos + 2 * nd]; pos += 2 * nd
        out.append({"mode": mode, "n_states": ns, "first": lo | (hi << 32), "bytes": bytes_, "table": table, "group": group, "desc": desc})
    assert pos == len(flat)
    return out


def _live_sets(seed, msg):
    """masks[j] = live states after message byte j (position j + 1 of the circuit); the device op's loop.
    Compact shape (mode 1): one state per position, masks[j] = 1 << (product that fires at byte j), 0 if none."""
    masks, mask = [], seed["first"]
    if seed["mode"] == 1:
        q = seed["first"]
        for c in msg:
            c = c if c < 255 else 255
            g, d = seed["group"][256 * q + c], seed["table"][256 * q + c]
            masks.append(0 if g == 0xff else 1 << g)
            q = 0 if d == 0xff else d
        return masks
    for c in msg:
        c = c if c < 255 else 255
        nxt = 1
        for s in range(seed["n_states"]):
            if (mask >> s) & 1:
                d = seed["table"][256 * s + c]
                if d != 0xff:
                    nxt |= 1 << d
        mask = nxt
        masks.append(mask)
    return masks


def _check(circuit, inputs, msg_of_seed):
    w = oracle_witness(circuit, inputs)
    seeds = _seeds(circuit)
    assert len(seeds) == len(msg_of_seed)
    total = 0
    for seed, msg in zip(seeds, msg_of_seed):
        assert [w[v] for v in seed["bytes"]] == list(msg)              # the recorded byte signals are the message
        masks = _live_sets(seed, msg)
        desc = seed["desc"]
        assert len(desc) > 0 and all(seed["table"][256 * s + 255] == 0xff for s in range(seed["n_states"]))
        for k in range(0, len(desc), 2):
            var, pos, st = desc[k], desc[k + 1] >> 8, desc[k + 1] & 0xff
            assert 1 <= pos <= len(msg) and (seed["mode"] == 1 or 1 <= st < seed["n_states"])
            assert w[var] == (masks[pos - 1] >> st) & 1, (pos, st)
        total += len(desc) // 2
    return total


def test_body_hash_regex_seed_table():
    c = z.Circuit("BodyHashRegex", [128, 0])
    hdr = b"to:a@b.c\r\ndkim-signature:v=1; a=rsa-sha256; bh=7xQMDuoVVU4m0W0WRVSrVXMeGSIASsnucK9dJsrc+vU=; h=from:to; b="
    rng = random.Random(3)
    alphabet = b"dkim-signature:bh=; \r\nazAZ09+/v\xc3\xa4\xff\x00"
    cases = [hdr, b"", b"\xff" * 5 + hdr[:60]] + [bytes(rng.choice(alphabet) for _ in range(rng.randrange(1, 128))) for _ in range(6)]
    for msg in cases:
        padded = list(msg) + [0] * (128 - len(msg))
        if any(b == 255 for b in padded):
            continue                                   # 255 is the marker byte: not a valid message byte for this circuit
        assert _check(c, {"msg": padded}, [padded]) > 1000


def test_compact_shape_seed_table():
    """The compact shape carries ONE one-hot state per position; its chain runs through the `fire` products (mode 1)."""
    c = z.Circuit("BodyHashRegex", [128, 1])
    assert [sd["mode"] for sd in _seeds(c)] == [1]
    hdr = b"to:a@b.c\r\ndkim-signature:v=1; a=rsa-sha256; bh=7xQMDuoVVU4m0W0WRVSrVXMeGSIASsnucK9dJsrc+vU=; h=from:to; b="
    rng = random.Random(5)
    alphabet = b"dkim-signature:bh=; \r\nazAZ09+/v\xc3\xa4\x00"
    for msg in [hdr, b"", b"dkim-signature:v=1; d=x; bh=QUJD; b="] + [bytes(rng.choice(alphabet) for _ in range(rng.randrange(1, 128))) for _ in range(6)]:
        padded = list(msg) + [0] * (128 - len(msg))
        assert _check(c, {"msg": padded}, [padded]) > 1000


def test_email_verifier_seed_table_on_a_signed_email():
    c = z.Circuit("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1])
    key = z.synthetic.generate_key()
    email = z.synthetic.make_signed_email(0, key, body_len=512)
    dk = z.verify_dkim_signature(email, resolver=lambda n, t: [z.synthetic.key_record(key)])
    inputs = z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": 640, "maxBodyLength": 768})
    header = [int(x) for x in inputs["emailHeader"]]
    assert _check(c, inputs, [header]) > 10000
