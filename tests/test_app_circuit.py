"""Email app circuits built from a spec (Circuit.from_spec, zke_circuit_build_app): EmailVerifier plus the app's own
regexes, revealed substrings and public inputs, as the zk-email usage guide has apps write by hand
(docs/zk-email-docs/UsageGuide/README.md, steps 1-2; Proof-of-Twitter is its worked example).  CPU only: witnesses come
from the oracle, which also checks every constraint.  The seeding of regexes with 65..255 DFA states (the wide mode of
witness.cu: regex_coop) is checked here on the host lowering; tests/test_gpu_app_circuit.py runs it on the device."""
import copy
import ctypes
import json
import random

import pytest

import zkemail_b200 as z
from zkutil import AssertFailed, oracle_witness

TWITTER_SPEC = {
    "maxHeadersLength": 1024, "maxBodyLength": 1536, "n": 121, "k": 17, "exposeHeaderHash": False,
    "regexes": [{"name": "twitterUsername", "location": "body",
                 "parts": [{"regexDef": "email was meant for @"},
                           {"regexDef": "[a-zA-Z0-9_]+", "isPublic": True, "maxLength": 21}]}],
    "externalInputs": [{"name": "address"}],
}

SENDER_DOMAIN = [("from:[^\r\n]*@", False), ("(gmail\\.com|icloud\\.com|outlook\\.com|yahoo\\.com|proton\\.me)", True)]
SUBJECT_MONTH = [("subject:[^\r\n]*", False),
                 ("(january|february|march|april|may|june|july|august|september|october|november|december)", True),
                 (" [0-9]+", False)]


def app_spec(style: int) -> dict:
    """The multi-regex app at EmailVerifier(640, 768): header from-address (zk-email's shape), the subject line, a body
    regex with two public parts, the sender-domain regex (74 DFA states: the wide seeding mode), a string external input and the email nullifier."""
    return {
        "maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": style,
        "regexes": [
            {"name": "fromAddress", "location": "header",
             "parts": [{"regexDef": "(\r\n|^)from:"}, {"regexDef": "([^\r\n]+<)?"},
                       {"regexDef": "[a-zA-Z0-9._%+-]+@[a-zA-Z0-9.-]+", "isPublic": True, "maxLength": 64},
                       {"regexDef": ">?\r\n"}]},
            {"name": "subject", "location": "header",
             "parts": [{"regexDef": "(\r\n|^)subject:"}, {"regexDef": "[^\r\n]+", "isPublic": True, "maxLength": 64},
                       {"regexDef": "\r\n"}]},
            {"name": "order", "location": "body",
             "parts": [{"regexDef": "Order #"}, {"regexDef": "[0-9]+", "isPublic": True, "maxLength": 10},
                       {"regexDef": " shipped to "}, {"regexDef": "[A-Za-z]+", "isPublic": True, "maxLength": 20}]},
            {"name": "senderDomain", "location": "header",
             "parts": [{"regexDef": SENDER_DOMAIN[0][0]}, {"regexDef": SENDER_DOMAIN[1][0], "isPublic": True, "maxLength": 31}]},
        ],
        "externalInputs": [{"name": "recipient", "maxLength": 42}],
        "emailNullifier": True,
    }


RECIPIENT = "0x71C7656EC7ab88b098defB751B7401B5f6d8976F"
SUBJECT = "Your order of 3 books"


def signed_app_email(index: int = 3, body_marker: str = "Order #40213 shipped to Alice"):
    key = z.synthetic.generate_key(seed=77)
    em = z.synthetic.make_signed_email(index, key, body_len=512, domain="gmail.com", marker=body_marker, subject=SUBJECT)
    return z.verify_dkim_signature(em, resolver=lambda n, t: [z.synthetic.key_record(key)])


EXPECTED = {"fromAddress": "sender0003@gmail.com", "subject": SUBJECT, "order0": "40213", "order1": "Alice",
            "senderDomain": "gmail.com", "recipient": RECIPIENT}

# stream digests of the existing circuits, recorded before the app builder and the wide seeding mode existed:
# (template, params) -> digest of zke_circuit_program_stats at cluster 1, 2 and 8
PINNED = {
    ("EmailVerifier", (640, 768, 121, 17, 0, 0, 0, 0, 0, 0)): ("4d76d1c12bc87b6e", "b35a05fc82b08041", "57c58a72a9bbb4e3"),
    ("EmailVerifier", (640, 768, 121, 17, 0, 0, 0, 0, 0, 1)): ("5528105d37e77396", "2398d7a6f361a4b1", "3b5d8408b05418bc"),
    ("TwitterVerifier", (1024, 1536, 121, 17, 0)): ("0d3470de1ecd01e8", "748eec9ef541096d", "d4c12c3b93a8126b"),
    ("TwitterVerifier", (1024, 1536, 121, 17, 1)): ("4620afe6819bba1a", "3a446aa987685934", "15c3681b3dd3a9d4"),
    ("BodyHashRegex", (256, 0)): ("07b129562fd77490", "6a01175a638d0928", "988f2bf70ae183d7"),
    ("BodyHashRegex", (256, 1)): ("9aecbcee4fedea7a", "96b5c6e69b9081c3", "040ae381d495de42"),
}


@pytest.mark.parametrize("template,params", list(PINNED), ids=[f"{t}-{p[-1]}" for t, p in PINNED])
def test_existing_streams_unchanged(template, params):
    c = z.Circuit(template, list(params))
    got = tuple("%016x" % c.program_stats(cluster=cl)["digest"] for cl in (1, 2, 8))
    assert got == PINNED[(template, params)]


def _same_circuit(a, b):
    assert a.write_r1cs() == b.write_r1cs()
    assert a.groups == b.groups
    for cl in (1, 8):
        assert a.program_stats(cluster=cl)["digest"] == b.program_stats(cluster=cl)["digest"]


@pytest.mark.parametrize("style", [0, 1])
def test_twitter_spec_is_twitter_verifier(style):
    spec = dict(TWITTER_SPEC, regexStyle=style)
    _same_circuit(z.Circuit.from_spec(spec), z.Circuit("TwitterVerifier", [1024, 1536, 121, 17, style]))
    _same_circuit(z.Circuit.from_spec(json.dumps(spec)), z.Circuit("TwitterVerifier", [1024, 1536, 121, 17, style]))


EV_FLAG_SETS = {
    "default": ({}, [0, 0, 0, 0, 0]),
    "masking": ({"enableHeaderMasking": True, "enableBodyMasking": True}, [0, 1, 1, 0, 0]),
    "soft_line_breaks": ({"removeSoftLineBreaks": True}, [0, 0, 0, 1, 0]),
    "ignore_body": ({"ignoreBodyHashCheck": True}, [1, 0, 0, 0, 0]),
    "public_pubkey": ({"publicPubkey": True}, [0, 0, 0, 0, 1]),
}


@pytest.mark.parametrize("flags", list(EV_FLAG_SETS))
def test_empty_spec_is_email_verifier(flags):
    extra, params = EV_FLAG_SETS[flags]
    spec = dict({"maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": 1}, **extra)
    _same_circuit(z.Circuit.from_spec(spec), z.Circuit("EmailVerifier", [640, 768, 121, 17] + params + [1]))


@pytest.fixture(scope="module", params=[0, 1], ids=["zkregex", "compact"])
def app(request):
    spec = app_spec(request.param)
    c = z.Circuit.from_spec(spec)
    inputs = z.generate_app_inputs(signed_app_email(), spec, {"recipient": RECIPIENT})
    return spec, c, inputs


def test_app_signal_layout(app):
    spec, c, _ = app
    outs = [g for g, (_, _, kind) in c.groups.items() if kind == 0]
    pubs = [g for g, (_, _, kind) in c.groups.items() if kind == 1]
    assert outs == ["pubkeyHash", "shaHi", "shaLo", "fromAddress", "subject", "order0", "order1", "senderDomain", "emailNullifier"]
    assert pubs == ["recipient"]
    assert list(c.groups)[-5:] == ["fromAddressIndex", "subjectIndex", "order0Index", "order1Index", "senderDomainIndex"]
    assert [c.groups[n][1] for n in ("fromAddress", "subject", "order0", "order1", "senderDomain", "recipient")] == [3, 3, 1, 1, 1, 2]


def test_app_witness_and_outputs(app):
    spec, c, inputs = app
    w = oracle_witness(c, inputs)                                    # checks every constraint
    publics = [w[1 + i] for i in range(c.info.n_public)]
    out = z.decode_app_outputs(spec, publics)
    assert {k: out[k] for k in EXPECTED} == EXPECTED
    assert out["pubkeyHash"] == w.values("pubkeyHash")[0] != 0 and out["emailNullifier"] != 0
    # the captures of Python's `re` on the same arrays are what the circuit reveals
    header = bytes(int(x) for x in inputs["emailHeader"])
    assert header[int(inputs["senderDomainIndex"]):].startswith(b"gmail.com")
    assert header[int(inputs["fromAddressIndex"]):].startswith(b"sender0003@gmail.com\r\n")


def test_app_rejects_bad_witnesses(app):
    spec, c, inputs = app
    for name in ("subjectIndex", "order1Index", "senderDomainIndex"):
        bad = dict(inputs, **{name: str(int(inputs[name]) + 1)})
        with pytest.raises(AssertFailed):
            oracle_witness(c, bad)
    # an email the sender-domain regex does not match
    dk = signed_app_email()
    other = z.synthetic.make_signed_email(3, z.synthetic.generate_key(seed=77), body_len=512, domain="example.com",
                                          marker="Order #40213 shipped to Alice", subject=SUBJECT)
    with pytest.raises(ValueError, match="senderDomain"):
        z.generate_app_inputs(other, spec, {"recipient": RECIPIENT},
                              {"resolver": lambda n, t: [z.synthetic.key_record(z.synthetic.generate_key(seed=77))]})
    spec_wo = copy.deepcopy(spec)
    spec_wo["regexes"] = [r for r in spec_wo["regexes"] if r["name"] != "senderDomain"]
    dko = z.verify_dkim_signature(other, resolver=lambda n, t: [z.synthetic.key_record(z.synthetic.generate_key(seed=77))])
    forced = z.generate_app_inputs(dko, spec_wo, {"recipient": RECIPIENT})
    forced["senderDomainIndex"] = inputs["senderDomainIndex"]
    with pytest.raises(AssertFailed):
        oracle_witness(c, forced)
    assert dk.headers != dko.headers


def test_non_ascii_regex_literal():
    """A regex literal outside ASCII is matched on its UTF-8 bytes by the circuit (the spec is JSON) and by the start-index
    search of generate_app_inputs alike."""
    spec = {"maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": 1,
            "regexes": [{"name": "ticket", "location": "body",
                         "parts": [{"regexDef": "Café 日 #"}, {"regexDef": "[0-9]+", "isPublic": True, "maxLength": 8}]}]}
    c = z.Circuit.from_spec(spec)
    inputs = z.generate_app_inputs(signed_app_email(5, "Réservation au Café 日 #7781 ok"), spec)
    body = bytes(int(x) for x in inputs["emailBody"])
    assert body[int(inputs["ticketIndex"]) - len("Café 日 #".encode()):].startswith("Café 日 #7781".encode())
    w = oracle_witness(c, inputs)
    assert z.decode_app_outputs(spec, [w[1 + i] for i in range(c.info.n_public)])["ticket"] == "7781"


def _refused(spec, *needles):
    with pytest.raises(z._lib.ZkeError) as e:
        z.Circuit.from_spec(spec)
    for n in needles:
        assert n in str(e.value), str(e.value)


def test_refusals():
    base = {"maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": 1}
    rx = lambda name, loc="header", parts=None: {"name": name, "location": loc, "parts": parts or [
        {"regexDef": "(\r\n|^)subject:"}, {"regexDef": "[^\r\n]+", "isPublic": True, "maxLength": 32}]}
    _refused(dict(base, colour=1), "spec", "unknown key 'colour'")
    _refused(dict(base, regexes=[dict(rx("a"), flags=1)]), "regexes[0]", "unknown key 'flags'")
    _refused(dict(base, regexes=[rx("a", loc="footer")]), "regexes[0].location", "footer")
    _refused(dict(base, regexes=[rx("a", parts=[{"regexDef": "x", "public": True}])]), "regexes[0].parts[0]", "unknown key 'public'")
    _refused(dict(base, externalInputs=[{"name": "x", "size": 3}]), "externalInputs[0]", "unknown key 'size'")
    _refused(dict(base, regexes=[rx("a"), rx("a")]), "regexes[1].name", "'a'", "used twice")
    _refused(dict(base, regexes=[rx("a")], externalInputs=[{"name": "aIndex"}]), "externalInputs[0].name", "'aIndex'")
    _refused(dict(base, regexes=[rx("signature")]), "regexes[0].name", "'signature'", "EmailVerifier signal")
    _refused(dict(base, externalInputs=[{"name": "pubkeyHash"}]), "externalInputs[0].name", "EmailVerifier signal")
    _refused(dict(base, externalInputs=[{"name": "x", "maxLength": 4200000000}]), "externalInputs[0].maxLength", "non-negative integer")
    _refused(dict(base, externalInputs=[{"name": "x", "maxLength": 65537}]), "externalInputs[0].maxLength", "at most 65536 bytes")
    _refused(dict(base, externalInputs=[{"name": "x", "maxLength": 0}]), "externalInputs[0].maxLength", "must be positive")
    _refused(dict(base, regexes=[rx("a", parts=[{"regexDef": "x"}, {"regexDef": "[a-z]+", "isPublic": True}])]),
             "regexes[0].parts[1].maxLength", "needs maxLength")
    _refused(dict(base, regexes=[rx("a", parts=[{"regexDef": "x"}, {"regexDef": "[a-z]+", "isPublic": True, "maxLength": 641}])]),
             "regexes[0].parts[1].maxLength", "larger than the searched header")
    _refused(dict(base, ignoreBodyHashCheck=True, regexes=[rx("a", loc="body")]), "regexes[0].location", "ignoreBodyHashCheck")
    _refused(dict(base, regexes=[rx("a", parts=[{"regexDef": "x*", "isPublic": True, "maxLength": 4}])]),
             "regexes[0] (a)", "matches the empty string")
    _refused(dict(base, regexes=[rx("a", parts=[{"regexDef": "x" * 700}])]), "regexes[0] (a)", "accept state unreachable")
    # no regexes and no external inputs: EmailVerifier alone
    assert z.Circuit.from_spec(base).info.n_public == 3


# The wide seeding mode on inputs that exercise it: for each regex a trigger string and the bytes of it after which a state
# >= 64 (words 1-3 of the live set) is live.  The messages place a trigger across every chunk boundary of the device run
# (witness.cu: regex_coop holds RX_CHUNK / 4 = 224 positions per chunk in the wide mode), each at a different hot byte, so
# the carry of the upper words and the upper-word reads of later chunks see non-zero values.
WIDE_CHUNK = 224
WIDE_CASES = {
    "sender_domain": (SENDER_DOMAIN, b"from:q@outlook.com ", range(15, 18), b"from:@gmailcom.icloudoutlkyahprtne \r\n"),
    "subject_month": (SUBJECT_MONTH, b"subject:x september 12 ", range(13, 22), b"subject:januryfebmchpilgstocvd 0123456789\r\n"),
}


def wide_regex_messages(case: str, n: int = 1024, count: int = 4, seed: int = 5):
    """`count` messages of n bytes: random bytes of the regex's alphabet with UTF-8 sequences and other bytes >= 0x80 mixed
    in, a trigger ending on a hot byte at every chunk boundary, more triggers in between, 40 zero bytes at the end."""
    _, trig, hot, alphabet = WIDE_CASES[case]
    hot = list(hot)
    rng = random.Random(seed)
    out = []
    for k in range(count):
        s = bytearray(rng.choice(alphabet) for _ in range(n - 40))
        for i in range(0, n - 60, 29):
            if rng.random() < 0.3:
                s[i:i + 3] = rng.choice(["é".encode() + b"x", "日".encode(), b"\x80\xc3\xfe"])
            elif rng.random() < 0.2:
                piece = trig[:rng.randrange(4, len(trig) + 1)]
                s[i:i + len(piece)] = piece
        for q, b in enumerate(range(WIDE_CHUNK, n - 40, WIDE_CHUNK)):
            j = hot[(k + q) % len(hot)]
            s[b - 1 - j:b - 1 - j + len(trig)] = trig          # its hot byte j is the last byte of the chunk
        assert len(s) == n - 40
        out.append(list(s) + [0] * 40)
    return out


def seed_records(c):
    """The flat seed image (ZKE_ARR_REGEX_SEEDS, include/zkemail_b200.h), narrow and wide records."""
    L = z._lib
    n = L.c_size_t()
    p = L.zke_circuit_array(c.handle, L.ARR_REGEX_SEEDS, ctypes.byref(n))
    flat = list((ctypes.c_uint32 * n.value).from_address(p)) if n.value else [0]
    out, pos = [], 1
    unpack = lambda words: [(wd >> (8 * k)) & 0xff for wd in words for k in range(4)]
    for _ in range(flat[0]):
        nd, nb, word = flat[pos:pos + 3]
        ns, wide, mode = word & 0x3fffffff, (word >> 30) & 1, word >> 31
        nf = 4 if wide else 1
        first = sum((flat[pos + 3 + 2 * q] | flat[pos + 4 + 2 * q] << 32) << (64 * q) for q in range(nf))
        pos += 3 + 2 * nf
        bytes_ = flat[pos:pos + nb]; pos += nb
        table = unpack(flat[pos:pos + 64 * ns]); pos += 64 * ns * (1 + mode)
        desc = flat[pos:pos + 2 * nd]; pos += 2 * nd
        out.append({"n_states": ns, "wide": wide, "mode": mode, "first": first, "bytes": bytes_, "table": table, "desc": desc})
    assert pos == len(flat)
    return out


def live_sets(seed, msg):
    """Live-state sets after each message byte: the device op's loop (zk-regex shape), as Python integers."""
    masks, mask = [], seed["first"]
    for c in msg:
        nxt = 1
        for s in range(seed["n_states"]):
            if (mask >> s) & 1:
                d = seed["table"][256 * s + min(c, 255)]
                if d != 0xff:
                    nxt |= 1 << d
        mask = nxt
        masks.append(mask)
    return masks


@pytest.mark.parametrize("case", list(WIDE_CASES))
def test_wide_regexes_are_seeded(case, monkeypatch):
    monkeypatch.setenv("ZKE_REGEX_STYLE", "0")
    c = z.Circuit.from_regex(WIDE_CASES[case][0], 1024)
    seeds = seed_records(c)
    assert len(seeds) == 1 and 64 < seeds[0]["n_states"] <= 255 and (seeds[0]["wide"], seeds[0]["mode"]) == (1, 0)
    st = c.program_stats()
    assert st["n_levels"] <= 16 and st["n_coop_ops"] == 1
    assert c.program_stats(native_regex=False)["n_levels"] > 6000


@pytest.mark.parametrize("case", list(WIDE_CASES))
def test_wide_seed_record_matches_oracle(case, monkeypatch):
    """Every seeded signal of a wide record holds its state's bit of the live set a Python run of the recorded table reaches
    (the values the device writes), and the messages the GPU test uses keep states >= 64 live across chunk boundaries."""
    monkeypatch.setenv("ZKE_REGEX_STYLE", "0")
    c = z.Circuit.from_regex(WIDE_CASES[case][0], 1024)
    seed = seed_records(c)[0]
    assert all(seed["table"][256 * s + 255] == 0xff for s in range(seed["n_states"]))
    carried = upper_reads = 0
    for msg in wide_regex_messages(case):
        w = oracle_witness(c, {"msg": msg})
        assert [w[v] for v in seed["bytes"]] == msg
        masks = live_sets(seed, msg)
        desc = seed["desc"]
        for k in range(0, len(desc), 2):
            var, pos, st = desc[k], desc[k + 1] >> 8, desc[k + 1] & 0xff
            assert 1 <= pos <= len(msg) and 1 <= st < seed["n_states"]
            assert w[var] == (masks[pos - 1] >> st) & 1, (pos, st)
            upper_reads += st >= 64 and pos > WIDE_CHUNK and w[var] == 1
        carried += sum(1 for b in range(WIDE_CHUNK, len(msg), WIDE_CHUNK) if masks[b - 1] >> 64)
        assert max(bin(m).count("1") for m in masks) >= 3                  # several states live at once
    assert carried >= 12 and upper_reads >= 12


CHUNK = 896                  # witness.cu: RX_CHUNK, positions per pass of the 64-state and compact seeding
LONG_REGEX = [("<", False), ("abcdefghijklmnopqrstuvwxyz0123456789ABCDEFGH", True), (">", False)]
LONG_LEN = 2000              # crosses the chunk boundaries at positions 896 and 1792
NON_BYTE = 256 + 7


def long_regex_messages(count: int = 3, seed: int = 11):
    """`count` messages of LONG_LEN bytes plus one that fails.  At every chunk boundary a match of LONG_REGEX is 32 to 43
    bytes into its literal (deep DFA states live in the carried set), with bytes >= 0x80 just before it and just after
    it; in the last message the match at the second boundary breaks on a byte >= 0x80 right after the boundary.  The
    extra message is the first one with a non-byte value just past the first boundary."""
    lit = LONG_REGEX[1][0].encode()
    rng = random.Random(seed)
    alphabet = b"<>abcxyz019ABCD \r\n"
    out = []
    for k in range(count):
        s = bytearray(rng.choice(alphabet) for _ in range(LONG_LEN))
        for q, b in enumerate(range(CHUNK, LONG_LEN, CHUNK)):
            depth = 32 + (5 * k + 3 * q) % (len(lit) - 32)       # literal bytes read by the end of the chunk
            start = b - depth - 1                                  # the '<'
            s[start - 2:start] = "é".encode()
            s[start:start + 2 + len(lit)] = b"<" + lit + b">"
            s[start + 2 + len(lit):start + 5 + len(lit)] = "日".encode()
            if k == count - 1 and q == 1:
                s[b] = 0xe9
        out.append(list(s))
    bad = list(out[0])
    bad[CHUNK] = NON_BYTE
    return out + [bad]


def _carried_states(seed, msg):
    """Per message byte, what the seeding carries to the next byte: the live-state mask (64-state shape) or the one live
    state (compact shape)."""
    if seed["mode"] == 0:
        return live_sets(seed, msg)
    q, out = seed["first"], []
    for c in msg:
        d = seed["table"][256 * q + min(c, 255)]
        q = 0 if d == 0xff else d
        out.append(q)
    return out


@pytest.mark.parametrize("style", [0, 1], ids=["zkregex", "compact"])
def test_long_regex_messages_cross_chunk_boundaries(style, monkeypatch):
    """The seeded signals of the messages tests/test_gpu_witness_edges.py runs hold the values a Python run of the recorded
    table gives, and at both chunk boundaries those messages carry a state >= 32 (the high half of the 64-bit mask, or a
    compact state number >= 32) into the next chunk, with bytes >= 0x80 within 16 bytes of the boundary."""
    from test_regex_seed_table import _check, _seeds
    monkeypatch.setenv("ZKE_REGEX_STYLE", str(style))
    c = z.Circuit.from_regex(LONG_REGEX, LONG_LEN)
    seeds = _seeds(c)
    assert len(seeds) == 1 and seeds[0]["mode"] == style and 32 < seeds[0]["n_states"] <= 64
    msgs = long_regex_messages()
    for msg in msgs[:-1]:
        assert _check(c, {"msg": msg}, [msg]) > LONG_LEN
        carried = _carried_states(seeds[0], msg)
        for b in range(CHUNK, LONG_LEN, CHUNK):
            assert (carried[b - 1] >> 32 if style == 0 else carried[b - 1] >= 32), (b, carried[b - 1])
            assert any(x >= 0x80 for x in msg[b - 16:b + 16])
    # a non-byte value fires no transition, as the marker 255 does; the zk-regex shape does not range-check its message,
    # the compact shape does
    bad = msgs[-1]
    assert bad[CHUNK] == NON_BYTE and bad[:CHUNK] == msgs[0][:CHUNK]
    if style == 0:
        assert _check(c, {"msg": bad}, [bad]) > LONG_LEN
    else:
        with pytest.raises(AssertFailed, match="Num2Bits"):
            oracle_witness(c, {"msg": bad})


def test_more_than_255_states_stay_unseeded(monkeypatch):
    monkeypatch.setenv("ZKE_REGEX_STYLE", "0")
    c = z.Circuit.from_regex([("x", False), ("[a-z]" * 300, True)], 320)
    assert seed_records(c) == []
    assert c.program_stats()["n_levels"] > 300                  # one chained level per byte at least
