"""Inputs and outputs of email app circuits (Circuit.from_spec; the builder is zke_circuit_build_app).

An app spec describes the circuit a zk-email app otherwise writes by hand (docs/zk-email-docs/UsageGuide/README.md: write
the regex, wrap EmailVerifier, reveal what it matched as public outputs):

    {"maxHeadersLength": 1024, "maxBodyLength": 1536, "n": 121, "k": 17,          # EmailVerifier and its flags
     "ignoreBodyHashCheck": false, "enableHeaderMasking": false, "enableBodyMasking": false,
     "removeSoftLineBreaks": false, "publicPubkey": false, "regexStyle": 1,
     "exposeHeaderHash": true,                        # shaHi / shaLo as outputs
     "shaPrecomputeSelector": "...",                  # input generation only
     "regexes": [{"name": "twitterUsername", "location": "body",
                  "parts": [{"regexDef": "email was meant for @"},
                            {"regexDef": "[a-zA-Z0-9_]+", "isPublic": true, "maxLength": 21}]}],
     "externalInputs": [{"name": "address"}, {"name": "note", "maxLength": 40}],
     "emailNullifier": false}

Every public part of a regex becomes a PackRegexReveal output of ceil(maxLength / 31) field elements, named after the
regex (`name`, or `name0`, `name1`, ... when the regex has several public parts), with a private start-index input
(`nameIndex` / `name0Index`, ...).

A public part may instead publish a hash of what it matched, with `"reveal"`:

    {"regexDef": "[a-z0-9.]+@[a-z0-9.]+", "isPublic": true, "maxLength": 64, "reveal": "hash"}
        one output: PoseidonModular(PackBytes(part, maxLength)) - poseidon_modular(pack_bytes(part, maxLength))
    {"regexDef": "...", "isPublic": true, "maxLength": 64, "reveal": "commit", "salt": "senderSalt"}
        one output: Poseidon(2)([that hash, salt]), the salt a private external input {"name": "senderSalt", "isPublic": false}

`"reveal": "bytes"` is the default.  External inputs are public unless `"isPublic": false`; private ones come after the
start indices in the witness.  expected_app_output gives the value a verifier compares an output with.

`"keyRegistryDepth": d` (1..32) hides the signing key too: the first output is then `registryRoot`, the root of a
KeyRegistry (registry.py) that holds the key's pubkeyHash, instead of pubkeyHash itself.  generate_app_inputs takes the
registry as params={"registry": reg} and fills the private inputs registryIndex and registrySiblings.

`"keyDomain": "<output name of a public header part>"` (with keyRegistryDepth, maxLength <= 255) binds the registry leaf to
a domain: the leaf is Poseidon(2)([domain_hash(D), pubkeyHash]) for the bytes D that part matched, so the registry must be
built with KeyRegistry.build_domains from (domain, key) pairs, and registryRoot then proves "signed by a key the registry
lists for domain D".  D itself is published as the part's reveal mode says (bytes, hash or commit)."""
from __future__ import annotations
import re

from .constants import MAX_BODY_PADDED_BYTES, MAX_HEADER_PADDED_BYTES
from .dkim import DKIMVerificationResult, verify_dkim_signature
from .input_generators import generate_email_verifier_inputs_from_dkim_result

_EV_FLAGS = ("ignoreBodyHashCheck", "enableHeaderMasking", "enableBodyMasking", "removeSoftLineBreaks",
             "shaPrecomputeSelector", "maxHeadersLength", "maxBodyLength")


def _chunks(max_length: int) -> int:
    return (max_length + 30) // 31


def public_parts(regex: dict) -> list[tuple[int, str, int]]:
    """[(index of the part, output name, maxLength)] of a spec regex, in signal order."""
    pub = [(i, p) for i, p in enumerate(regex["parts"]) if p.get("isPublic")]
    name = regex["name"]
    return [(i, name if len(pub) == 1 else f"{name}{q}", int(p["maxLength"])) for q, (i, p) in enumerate(pub)]


def _reveal(regex: dict, index: int) -> str:
    return regex["parts"][index].get("reveal", "bytes")


def expected_app_output(spec: dict, name: str, value_bytes, salt=None) -> int | str:
    """The value the app output `name` holds when its part matched `value_bytes`: the string itself for a plain reveal,
    poseidon_modular(pack_bytes(value, maxLength)) for `"reveal": "hash"`, and Poseidon(2)([that hash, salt]) for
    `"reveal": "commit"` - what a verifier who knows the value (and the salt) compares the public signal with."""
    from .hash import poseidon, poseidon_modular
    data = value_bytes.encode("utf-8") if isinstance(value_bytes, str) else bytes(value_bytes)
    for rx in spec.get("regexes", []):
        for i, out, max_length in public_parts(rx):
            if out != name:
                continue
            mode = _reveal(rx, i)
            if mode == "bytes":
                return data.decode("utf-8", errors="replace")
            h = poseidon_modular(int(x) for x in pack_bytes(data, max_length))
            if mode == "hash":
                return h
            if salt is None:
                raise ValueError(f'output "{name}" is a commitment: the salt is needed')
            return poseidon([h, int(salt, 0) if isinstance(salt, str) else int(salt)])
    raise ValueError(f'the spec has no revealed part named "{name}"')


def pack_bytes(data: bytes, max_length: int) -> list[str]:
    """PackBytes(maxLength) of `data` zero-padded to maxLength: 31 bytes per field element, little-endian."""
    if len(data) > max_length:
        raise ValueError(f"{len(data)} bytes do not fit maxLength {max_length}")
    data = data + b"\0" * (max_length - len(data))
    return [str(int.from_bytes(data[31 * i:31 * i + 31], "little")) for i in range(_chunks(max_length))]


def unpack_bytes(values) -> bytes:
    out = b"".join(int(v).to_bytes(31, "little") for v in values)
    return out.rstrip(b"\0")


def _python_regex(parts) -> re.Pattern:
    """The decomposed regex as one Python pattern on bytes, each part a named group `p<i>`.  The dialect is the same
    subset (zk-regex's `^` is the start of the searched array, as in Python without MULTILINE; `.` matches newlines).
    Non-ASCII characters are matched as their UTF-8 bytes, as the circuit builder reads the spec's JSON strings."""
    return re.compile(b"".join(b"(?P<p%d>" % i + p["regexDef"].encode("utf-8") + b")" for i, p in enumerate(parts)), re.DOTALL)


def generate_app_inputs(raw_email_or_dkim_result, spec: dict, external_inputs: dict | None = None,
                        params: dict | None = None) -> dict:
    """Circuit inputs of an app circuit: the EmailVerifier inputs (with the spec's flags and shaPrecomputeSelector), the
    start index of every public part - found by running the same decomposed regex through Python `re` on the array the
    circuit searches (emailHeader, emailBody or decodedEmailBodyIn) - and the external inputs, private ones (salts)
    included (strings with a maxLength are packed, everything else is one field element).  `params` may add headerMask / bodyMask and, for a raw email, a
    DKIM key `resolver`.  Raises ValueError naming the regex that does not match."""
    params = dict(params or {})
    resolver = params.pop("resolver", None)
    registry = params.pop("registry", None)
    depth = int(spec.get("keyRegistryDepth", 0))
    if depth and registry is None:
        raise ValueError(f'the spec has "keyRegistryDepth": {depth}: pass params={{"registry": KeyRegistry}}')
    if depth and registry.depth != depth:
        raise ValueError(f"the registry has depth {registry.depth}, the spec keyRegistryDepth {depth}")
    key_domain = spec.get("keyDomain")
    if depth and bool(key_domain) != registry.domain_bound:
        raise ValueError(f'the spec has "keyDomain": {key_domain!r}: pass a registry of (domain, key) leaves '
                         '(KeyRegistry.build_domains)' if key_domain else
                         'the registry holds (domain, key) leaves: the spec needs "keyDomain"')
    domain = None
    if isinstance(raw_email_or_dkim_result, DKIMVerificationResult):
        dk = raw_email_or_dkim_result
    else:
        dk = verify_dkim_signature(raw_email_or_dkim_result, resolver=resolver)
    ev = {k: spec[k] for k in _EV_FLAGS if k in spec}
    ev.setdefault("maxHeadersLength", MAX_HEADER_PADDED_BYTES)
    ev.setdefault("maxBodyLength", MAX_BODY_PADDED_BYTES)
    ev.update(params)
    inputs = generate_email_verifier_inputs_from_dkim_result(dk, ev)
    for rx in spec.get("regexes", []):
        if rx["location"] == "header":
            arr = inputs["emailHeader"]
        else:
            arr = inputs["decodedEmailBodyIn" if spec.get("removeSoftLineBreaks") else "emailBody"]
        hay = bytes(int(x) for x in arr)
        m = _python_regex(rx["parts"]).search(hay)
        if m is None:
            raise ValueError(f'regex "{rx["name"]}" does not match the email\'s {rx["location"]}')
        for i, name, _ in public_parts(rx):
            inputs[name + "Index"] = str(m.start(f"p{i}"))
            if name == key_domain:
                domain = m.group(f"p{i}")
    external_inputs = external_inputs or {}
    for ei in spec.get("externalInputs", []):
        name = ei["name"]
        if name not in external_inputs:
            raise ValueError(f'external input "{name}" is missing')
        v = external_inputs[name]
        if "maxLength" in ei:
            data = v.encode() if isinstance(v, str) else bytes(v)
            inputs[name] = pack_bytes(data, int(ei["maxLength"]))
        else:
            inputs[name] = str(int(v, 0) if isinstance(v, str) else int(v))
    if depth:
        from .hash import canonical_domain, domain_words, poseidon, poseidon_large
        n, k = int(spec.get("n", 121)), int(spec.get("k", 17))
        leaf = poseidon_large(dk.publicKey, (k + 1) // 2, 2 * n)
        if key_domain:
            # the circuit hashes the matched bytes as they are: a name not in canonical form has no leaf in any registry
            text = domain.decode("utf-8", errors="replace")
            try:
                canonical = canonical_domain(domain) == domain
            except ValueError:
                canonical = False
            if not canonical:
                raise ValueError(f'{key_domain} "{text}" is not a canonical domain (lower-case ASCII, no trailing dot): '
                                 "no registry leaf can match it")
            leaf = poseidon([poseidon(domain_words(domain)), leaf])
            if leaf not in registry.leaves:
                raise ValueError(f'the signing key is not registered for domain "{text}"')
        index, siblings = registry.path(registry.index_of(leaf))
        inputs["registryIndex"] = str(index)
        inputs["registrySiblings"] = [str(x) for x in siblings]
    return inputs


def decode_app_outputs(spec: dict, public_signals) -> dict:
    """Public signals of an app proof (snarkjs public.json order) -> {name: value}: revealed substrings and packed
    external inputs as strings, every other signal as an int (hashed and committed parts included; the masks as lists of
    byte values).  Private external inputs are not public signals.  With keyRegistryDepth the first signal is
    registryRoot instead of pubkeyHash."""
    sig = [int(x) for x in public_signals]
    pos = 0

    def take(n):
        nonlocal pos
        if pos + n > len(sig):
            raise ValueError(f"{len(sig)} public signals are too few for this spec")
        pos += n
        return sig[pos - n:pos]

    H = int(spec.get("maxHeadersLength", MAX_HEADER_PADDED_BYTES))
    Bd = int(spec.get("maxBodyLength", MAX_BODY_PADDED_BYTES))
    out = {"registryRoot" if spec.get("keyRegistryDepth") else "pubkeyHash": take(1)[0]}
    if spec.get("exposeHeaderHash", True):
        out["shaHi"], out["shaLo"] = take(2)
    if spec.get("enableHeaderMasking"):
        out["maskedHeader"] = take(H)
    if not spec.get("ignoreBodyHashCheck") and spec.get("enableBodyMasking"):
        out["maskedBody"] = take(Bd)
    for rx in spec.get("regexes", []):
        for i, name, max_length in public_parts(rx):
            if _reveal(rx, i) == "bytes":
                out[name] = unpack_bytes(take(_chunks(max_length))).decode("utf-8", errors="replace")
            else:
                out[name] = take(1)[0]
    if spec.get("emailNullifier"):
        out["emailNullifier"] = take(1)[0]
    for ei in spec.get("externalInputs", []):
        if not ei.get("isPublic", True):
            continue
        if "maxLength" in ei:
            out[ei["name"]] = unpack_bytes(take(_chunks(int(ei["maxLength"])))).decode("utf-8", errors="replace")
        else:
            out[ei["name"]] = take(1)[0]
    if spec.get("publicPubkey"):
        out["pubkey"] = take(int(spec.get("k", 17)))
    if pos != len(sig):
        raise ValueError(f"{len(sig)} public signals, the spec accounts for {pos}")
    return out


__all__ = ["generate_app_inputs", "decode_app_outputs", "expected_app_output", "pack_bytes", "unpack_bytes", "public_parts"]
