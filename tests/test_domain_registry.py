"""Registry leaves bound to domains (`"keyDomain"` in a spec with `"keyRegistryDepth"`): the leaf is
Poseidon(2)([domainHash(D), pubkeyHash]) with domainHash(D) = PoseidonModular(PackBytes(D, 255)), D the bytes a public
header part matched, so registryRoot proves "signed by a key the registry lists for domain D".  CPU only: the leaf
against a restatement on oracle/poseidon.py, the canonical form of names, every spec refusal, the app circuit on the
oracle witness with D from a DKIM `d=` tag (revealed as bytes) and from the From address (committed), the Poseidon
records, the level and op counts, the negative cases, and the pinned circuit of a spec without keyDomain.
tests/test_gpu_domain_registry.py runs the GPU side."""
import copy
import ctypes
import hashlib

import pytest

import zkemail_b200 as z
from oracle import merkle
from oracle import poseidon as oracle_poseidon
from test_app_commit import SALT, commit_spec, permutation_signals, poseidon_records, signed_commit_email
from zkutil import AssertFailed, oracle_witness

R = z.FR_MODULUS
DEPTH = 4
DOMAIN_SALT = 0x5eed_d0_a1_2026


def oracle_domain_key_leaf(domain: bytes, modulus: int, n: int = 121, k: int = 17) -> int:
    """The leaf restated on the oracle's permutation: the name zero-padded to 255 bytes, 9 little-endian words of 31
    bytes, Poseidon(9); the modulus through PoseidonLarge; Poseidon(2) of the two."""
    row = domain.ljust(255, b"\0")
    words = [int.from_bytes(row[31 * i:31 * i + 31], "little") for i in range(9)]
    dh = oracle_poseidon.poseidon(words)
    return oracle_poseidon.poseidon([dh, oracle_poseidon.poseidon_large(modulus, (k + 1) // 2, 2 * n)])


# ---- the leaf --------------------------------------------------------------------------------------------------------

def _name(length: int) -> bytes:
    """A canonical name of `length` bytes: labels of seven characters, ending in a letter."""
    return (b"abc-de7." * 32)[:length - 1] + b"z"


@pytest.mark.parametrize("length", [1, 30, 31, 32, 62, 255])
def test_leaf_matches_oracle(length):
    d = _name(length)
    assert len(d) == length
    m = z.synthetic.generate_key(seed=77).public_key().public_numbers().n
    hash_spec = {"regexes": [{"name": "d", "location": "header",
                              "parts": [{"regexDef": "d="}, {"regexDef": "[a-z0-9.-]+", "isPublic": True, "maxLength": 255,
                                                             "reveal": "hash"}]}]}
    dh = z.hash.domain_hash(d.decode())
    assert dh == oracle_poseidon.poseidon_modular([int(x) for x in z.app.pack_bytes(d, 255)])
    assert dh == z.expected_app_output(hash_spec, "d", d)
    assert z.registry.domain_key_leaf(d.decode(), m) == oracle_domain_key_leaf(d, m)


def test_canonical_domain():
    assert z.hash.canonical_domain("Mail.Example.COM.") == b"mail.example.com"
    assert z.hash.domain_hash("GMAIL.com.") == z.hash.domain_hash("gmail.com")
    assert z.hash.canonical_domain("xn--bcher-kva.example") == b"xn--bcher-kva.example"
    for bad, needle in (("bücher.example", "A-label"), ("", "1 to 255"), (".", "1 to 255"), ("a" * 256, "1 to 255"),
                        ("a\0b", "zero byte"), (b"\xc3\xbc.de", "not ASCII")):
        with pytest.raises(ValueError, match=needle):
            z.hash.canonical_domain(bad)
        with pytest.raises(ValueError, match=needle):
            z.KeyRegistry.build_domains([(bad, 3)], 4)           # refused before any device is touched


# ---- specs -----------------------------------------------------------------------------------------------------------

def dkim_domain_regex(max_length: int = 64, reveal: str = "bytes") -> dict:
    return {"name": "dkimDomain", "location": "header",
            "parts": [{"regexDef": "(\r\n|^)dkim-signature:"}, {"regexDef": "([a-z]+=[^;]+; )+d="},
                      {"regexDef": "[a-z0-9.-]+", "isPublic": True, "maxLength": max_length, "reveal": reveal},
                      {"regexDef": ";"}]}


def from_domain_regex() -> dict:
    return {"name": "senderDomain", "location": "header",
            "parts": [{"regexDef": "(\r\n|^)from:"}, {"regexDef": "[^\r\n@]+@"},
                      {"regexDef": "[a-z0-9.-]+", "isPublic": True, "maxLength": 40, "reveal": "commit", "salt": "domainSalt"},
                      {"regexDef": "\r\n"}]}


def domain_spec(style: int, kind: str, bound: bool = True, depth: int = DEPTH) -> dict:
    """commit_spec with a registry and a domain part: the `d=` tag revealed as bytes, or the From domain committed."""
    spec = copy.deepcopy(commit_spec(style))
    spec["keyRegistryDepth"] = depth
    if kind == "dkim":
        spec["regexes"].append(dkim_domain_regex())
        name = "dkimDomain"
    else:
        spec["regexes"].append(from_domain_regex())
        spec["externalInputs"].append({"name": "domainSalt", "isPublic": False})
        name = "senderDomain"
    if bound:
        spec["keyDomain"] = name
    return spec


def email_modulus() -> int:
    return signed_commit_email().publicKey


N_PAIRS = 11
POSITION = 6


def oracle_registry(domain: bytes = b"gmail.com", depth: int = DEPTH) -> z.KeyRegistry:
    """N_PAIRS domain-bound leaves from the oracle: the email's key under `domain` at POSITION, the same key under other
    domains, and other keys under gmail.com."""
    m = email_modulus()
    leaves = [oracle_domain_key_leaf(b"other%d.example" % i, m) if i % 2 else oracle_domain_key_leaf(b"gmail.com", pow(3, 2000 + i) | 1)
              for i in range(N_PAIRS)]
    leaves[POSITION] = oracle_domain_key_leaf(domain, m)
    return z.KeyRegistry(depth, merkle.levels(leaves, depth), domain_bound=True)


def _externals(kind):
    ext = {"senderSalt": SALT, "recipient": 77}
    if kind == "from":
        ext["domainSalt"] = DOMAIN_SALT
    return ext


def _inputs(spec, kind, reg):
    return z.generate_app_inputs(signed_commit_email(), spec, _externals(kind), params={"registry": reg})


_APPS = {}


def _app(style, kind, bound=True):
    key = (style, kind, bound)
    if key not in _APPS:
        spec = domain_spec(style, kind, bound)
        _APPS[key] = (spec, z.Circuit.from_spec(spec))
    return _APPS[key]


KINDS = [(0, "dkim"), (1, "dkim"), (0, "from"), (1, "from")]
KIND_IDS = ["zkregex-dkim-bytes", "compact-dkim-bytes", "zkregex-from-commit", "compact-from-commit"]


@pytest.mark.parametrize("style,kind", KINDS, ids=KIND_IDS)
def test_app_domain_bound_root(style, kind):
    spec, c = _app(style, kind)
    reg = oracle_registry()
    inputs = _inputs(spec, kind, reg)
    assert inputs["registryIndex"] == str(POSITION)
    w = oracle_witness(c, inputs)                                   # checks every constraint
    out = z.decode_app_outputs(spec, [w[1 + i] for i in range(c.info.n_public)])
    assert out["registryRoot"] == merkle.root(reg.leaves, DEPTH) == reg.root
    if kind == "dkim":
        assert out["dkimDomain"] == "gmail.com"
    else:
        assert out["senderDomain"] == z.expected_app_output(spec, "senderDomain", "gmail.com", DOMAIN_SALT)
    leaf = oracle_domain_key_leaf(b"gmail.com", email_modulus())
    assert merkle.check_path(reg.root, leaf, POSITION, [int(x) for x in inputs["registrySiblings"]])
    # no signal of its own: the same groups as without keyDomain
    assert c.groups.keys() == _app(style, kind, False)[1].groups.keys()

    # the Poseidon records (the two leaf hashes among them) replay on the oracle witness
    blocks = poseidon_records(c)
    for b in blocks:
        vals = permutation_signals(b["t"], [0] + [w[v] for v in b["inputs"]])
        seen = set()
        for q in range(0, len(b["desc"]), 2):
            var, word = b["desc"][q], b["desc"][q + 1]
            assert w[var] == vals[(word >> 16, (word >> 8) & 0xff, word & 0xff)]
            seen.add(var)
        assert seen == set(range(*b["var"]))
    # after the app's hashes: Poseidon(9) of the domain (its padding words one repeated zero signal), the leaf, the path
    d9, lf = blocks[-2 - DEPTH], blocks[-1 - DEPTH]
    assert d9["t"] == 10 and lf["t"] == 3 and [b["t"] for b in blocks[-DEPTH:]] == [3] * DEPTH
    n_words = 3 if kind == "dkim" else 2                            # maxLength 64 / 40
    pad = d9["inputs"][n_words:]
    assert len(set(pad)) == 1 and w[pad[0]] == 0
    assert w[d9["desc"][-2]] == z.hash.domain_hash("gmail.com")
    assert lf["inputs"][0] == d9["desc"][-2]
    assert w[lf["desc"][-2]] == leaf
    if kind == "dkim":
        assert d9["inputs"][:n_words] == list(range(c.groups["dkimDomain"][0], c.groups["dkimDomain"][0] + n_words))


@pytest.mark.parametrize("style,kind", KINDS, ids=KIND_IDS)
def test_native_poseidon_ops_and_levels(style, kind):
    """Exactly two more native Poseidon ops than the same spec without keyDomain.  The leaf's two hashes and the path
    (three levels per tree level: swap product, left / right, node hash) now follow the domain's PackRegexReveal instead
    of running next to the regexes; at EmailVerifier(640, 768) and depth 4 that chain ends one level after the deepest
    chain of the app without it (355 against 354 levels at cluster widths 1 and 8, both regex shapes)."""
    spec, c = _app(style, kind)
    _, plain = _app(style, kind, False)
    for cl in (1, 8):
        on, base = c.program_stats(cluster=cl), plain.program_stats(cluster=cl)
        assert on["n_coop_ops"] - base["n_coop_ops"] == 2
        assert on["n_coop_ops"] - c.program_stats(cluster=cl, native_poseidon=False)["n_coop_ops"] == len(poseidon_records(c))
        assert on["n_levels"] - base["n_levels"] == 1, (on["n_levels"], base["n_levels"])


def test_shifted_domain_index_fails():
    spec, c = _app(1, "dkim")
    inputs = _inputs(spec, "dkim", oracle_registry())
    with pytest.raises(AssertFailed):
        oracle_witness(c, dict(inputs, dkimDomainIndex=str(int(inputs["dkimDomainIndex"]) + 1)))
    with pytest.raises(AssertFailed):
        oracle_witness(c, dict(inputs, dkimDomainIndex=str(int(inputs["dkimDomainIndex"]) - 1)))


def test_other_leaf_path_gives_other_root():
    spec, c = _app(1, "dkim")
    reg = oracle_registry()
    inputs = _inputs(spec, "dkim", reg)
    for other in (POSITION - 1, POSITION + 1):                      # the same key under another domain, another key
        index, sib = reg.path(other)
        w = oracle_witness(c, dict(inputs, registryIndex=str(index), registrySiblings=[str(x) for x in sib]))
        assert w.values("registryRoot")[0] != reg.root


def test_key_registered_for_another_domain():
    spec, _ = _app(1, "dkim")
    reg = oracle_registry(domain=b"yahoo.com")                      # the key under yahoo.com only, the email says gmail.com
    with pytest.raises(ValueError, match='domain "gmail.com"'):
        _inputs(spec, "dkim", reg)
    plain = z.KeyRegistry(DEPTH, merkle.levels([pow(7, 100 + i, R) for i in range(5)], DEPTH))
    with pytest.raises(ValueError, match="build_domains"):
        _inputs(spec, "dkim", plain)
    with pytest.raises(ValueError, match="keyDomain"):
        _inputs(domain_spec(1, "dkim", bound=False), "dkim", oracle_registry())


def test_registry_json_round_trip_marks_leaf():
    reg = oracle_registry()
    assert '"leaf": "domainKey"' in reg.to_json()
    plain = z.KeyRegistry(DEPTH, merkle.levels([1, 2, 3], DEPTH))
    assert "leaf" not in plain.to_json()
    with pytest.raises(ValueError, match="unknown registry leaf"):
        z.KeyRegistry.from_json('{"depth": 4, "leaves": ["1"], "leaf": "other"}')


# ---- refusals --------------------------------------------------------------------------------------------------------

def _refused(spec, *needles):
    with pytest.raises(z._lib.ZkeError) as e:
        z.Circuit.from_spec(spec)
    for n in needles:
        assert n in str(e.value), str(e.value)


def test_spec_refusals():
    base = {"maxHeadersLength": 640, "maxBodyLength": 768, "regexStyle": 1, "keyRegistryDepth": 3,
            "regexes": [dkim_domain_regex()], "externalInputs": [{"name": "ext"}]}
    z.Circuit.from_spec(dict(base, keyDomain="dkimDomain"))
    _refused(dict(base, keyDomain="dkimDomain", keyRegistryDepth=0), "keyDomain", "needs keyRegistryDepth")
    nodepth = dict(base, keyDomain="dkimDomain")
    del nodepth["keyRegistryDepth"]
    _refused(nodepth, "keyDomain", "needs keyRegistryDepth")
    _refused(dict(base, keyDomain="ext"), "keyDomain", "'ext'", "not the output name of a public regex part")
    _refused(dict(base, keyDomain="dkimDomainIndex"), "keyDomain", "not the output name of a public regex part")
    private = dict(base, regexes=[{"name": "hidden", "location": "header",
                                   "parts": [{"regexDef": "(\r\n|^)dkim-signature:"}, {"regexDef": "[^;]+"}]}])
    _refused(dict(private, keyDomain="hidden"), "keyDomain", "'hidden'", "not the output name of a public regex part")
    body = dict(base, regexes=[{"name": "bodyDomain", "location": "body",
                                "parts": [{"regexDef": "Domain: "}, {"regexDef": "[a-z.]+", "isPublic": True, "maxLength": 32}]}])
    _refused(dict(body, keyDomain="bodyDomain"), "keyDomain", "'bodyDomain'", "body regex part", "signed header")
    _refused(dict(base, regexes=[dkim_domain_regex(256)], keyDomain="dkimDomain"), "keyDomain", "maxLength 256", "at most 255")
    z.Circuit.from_spec(dict(base, regexes=[dkim_domain_regex(255, "hash")], keyDomain="dkimDomain"))
    _refused(dict(base, keyDomain=""), "keyDomain", "empty name")
    _refused(dict(base, keyDomain=3), "keyDomain", "expected a string")


def test_spec_without_key_domain_is_pinned():
    """The keyRegistryDepth spec of test_key_registry.py keeps its R1CS bytes and program digests (values of the commit
    before keyDomain existed)."""
    pinned = {0: ("dc9588bf05d902af9acc9715d3926cf4e4de0633dafde867b6b788ab8ae22cff", [4666624207938867228, 6883072847949192153]),
              1: ("9909ca5a22b92c2ee39a4fc6e441b435a15c21ff13dc505a11452e9fdcad9e04", [13365130502076658501, 14949766120579686067])}
    for style, (r1cs, digests) in pinned.items():
        c = z.Circuit.from_spec(dict(commit_spec(style), keyRegistryDepth=DEPTH))
        assert hashlib.sha256(c.write_r1cs()).hexdigest() == r1cs
        assert [c.program_stats(cluster=cl)["digest"] for cl in (1, 8)] == digests


def test_native_call_refuses_bad_arguments():
    """Argument checks come before the device: these refusals hold with or without a GPU."""
    L = z._lib
    err = ctypes.create_string_buffer(L.ERRCAP)
    out = ctypes.create_string_buffer(64)
    rows = b"gmail.com".ljust(255, b"\0")
    assert L.zke_domain_key_leaves(bytes(256), 1, 256, 121, 16, rows, 0, out, err, L.ERRCAP) < 0 and b"k must be 17..32" in err.value
    assert L.zke_domain_key_leaves(bytes(256), 1, 256, 126, 17, rows, 0, out, err, L.ERRCAP) < 0 and b"2n < 251" in err.value
    assert L.zke_domain_key_leaves(bytes(256), 1, 0, 121, 17, rows, 0, out, err, L.ERRCAP) < 0 and b"modulus_bytes" in err.value
    assert L.zke_domain_key_leaves(bytes(256), 1, 256, 121, 17, None, 0, out, err, L.ERRCAP) < 0 and b"null argument" in err.value
    assert L.zke_domain_key_leaves(bytes(256), 0, 256, 121, 17, rows, 0, out, err, L.ERRCAP) == 0
    if z.device_count() == 0:
        assert L.zke_domain_key_leaves(bytes(256), 1, 256, 121, 17, rows, 0, out, err, L.ERRCAP) < 0 and b"no CPU fallback" in err.value
