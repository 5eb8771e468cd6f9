"""Keys from a Powers-of-Tau file on the GPU (Zkey.from_ptau), phase-2 contributions (Zkey.contribute) and their check
(Zkey.check_contribution / verify_zkey), against the CPU oracle's setup and the seeded toy setup."""
import ctypes
import struct

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkutil import oracle_prove, oracle_setup, product_sections
from ptau_writer import R, write_ptau
from oracle import bn254

pytestmark = pytest.mark.gpu

TOX = (0x1F2E3D4C5B6A79880123456789ABCDEF0FEDCBA98765432, 0x2468ACE013579BDF2468ACE013579BDF, 0x0DDBA11CAFEBABE5EED)
S1, S2 = 0x5EC2E7 * 10 ** 30 + 17, 0xC0FFEE * 10 ** 25 + 3


def _le(x):
    return int(x).to_bytes(32, "little")


@pytest.fixture(scope="module")
def ptau14():
    return z.ptau_toy(14, *TOX)


def test_native_toy_writer_matches_python_writer():
    assert bytes(z.ptau_toy(2, *TOX)) == write_ptau(2, *TOX)[0]


@pytest.mark.parametrize("tmpl", [("SelectRegexReveal", [34, 8]), ("PackRegexReveal", [64, 21]), ("PoseidonModular", [37])])
def test_from_ptau_and_contributions_equal_the_oracle_setup(ptau14, tmpl):
    c = z.Circuit(*tmpl)
    base = z.Zkey.from_ptau(c, ptau14)
    assert base.is_toy
    assert product_sections(base) == oracle_setup(c, TOX + (1, 1)), "from_ptau differs from the oracle setup at gamma = delta = 1"
    k1 = base.contribute(_le(S1))
    assert not k1.is_toy
    assert product_sections(k1) == oracle_setup(c, TOX + (1, S1))
    k2 = k1.contribute(_le(S2))
    assert product_sections(k2) == product_sections(base.contribute(_le(S1 * S2 % R)))
    assert k1.check_contribution(base) and k2.check_contribution(k1) and k2.check_contribution(base)


def test_contribution_secrets_are_checked(ptau14):
    c = z.Circuit("SelectRegexReveal", [34, 8])
    base = z.Zkey.from_ptau(c, ptau14)
    for bad, msg in ((0, "zero"), (1, "one"), (R, "below the group order")):
        with pytest.raises(L.ZkeError, match=msg):
            base.contribute(_le(bad))
    assert not base.contribute().is_toy          # drawn from `secrets`
    seeded = z.Zkey(c, seed=3)
    assert seeded.contribute(_le(S1)).is_toy     # its tau is known: still a toy


# ------------------------------------------------------------------------------------------------ tampered keys
def _sections(data: bytes) -> dict:
    n = struct.unpack_from("<I", data, 8)[0]
    pos, out = 12, {}
    for _ in range(n):
        t, size = struct.unpack_from("<IQ", data, pos)
        out[t] = (pos + 12, size)
        pos += 12 + size
    return out


def _patched(key: z.Zkey, section: int, index: int, size: int, src_index: int) -> z.Zkey:
    """The key written to a `.zkey`, point `index` of `section` replaced by point `src_index` of the same section, loaded back."""
    data = bytearray(key.write())
    off = _sections(data)[section][0]
    data[off + size * index:off + size * (index + 1)] = data[off + size * src_index:off + size * (src_index + 1)]
    return z.Zkey.load(bytes(data), circuit=key.circuit)


def test_check_contribution_rejects_tampered_keys(ptau14):
    c = z.Circuit("PackRegexReveal", [64, 21])
    base = z.Zkey.from_ptau(c, ptau14)
    key = base.contribute(_le(S1)).contribute(_le(S2))
    ok, why = key.contribution_report(base)
    assert ok and why == ""
    assert z.verify_zkey(c, ptau14, key)
    loaded = z.Zkey.load(key.write(), circuit=c)
    assert loaded.check_contribution(base)
    def changing(sec, size):   # an index whose point differs from the next one
        pts = key.section(sec)
        return next(i for i in range(c.info.n_vars - 1) if pts[size * i:size * (i + 1)] != pts[size * (i + 1):size * (i + 2)])
    ja, jb = changing(L.SEC_A, 64), changing(L.SEC_B2, 128)
    cases = {
        "L point": (_patched(key, 8, 3, 64, 4), "L and H points"),
        "H point": (_patched(key, 9, 5, 64, 6), "L and H points"),
        "A point": (_patched(key, 5, ja, 64, ja + 1), f"A point {ja} differs"),
        "B2 point": (_patched(key, 7, jb, 128, jb + 1), f"B2 point {jb} differs"),
    }
    # delta1 (header offset 468) replaced by alpha1 (offset 84): a valid point with another discrete logarithm
    data = bytearray(key.write())
    h = _sections(data)[2][0]
    data[h + 468:h + 532] = data[h + 84:h + 148]
    cases["delta1"] = (z.Zkey.load(bytes(data), circuit=c), "different discrete logarithms")
    for name, (bad, reason) in cases.items():
        ok, why = bad.contribution_report(base)
        assert not ok, f"{name}: tampered key accepted"
        assert reason in why, f"{name}: {why}"
    other = z.Zkey.from_ptau(z.Circuit("SelectRegexReveal", [34, 8]), ptau14).contribute(_le(S1))
    ok, why = other.contribution_report(base)
    assert not ok and "different shapes" in why
    assert not z.verify_zkey(c, z.ptau_toy(12, TOX[0] + 1, TOX[1], TOX[2]), key)


# ------------------------------------------------------------------------------------------------ write / load / registry
def test_contributed_key_writes_loads_and_proves_identically(ptau14, tmp_path):
    import hashlib
    c = z.Circuit("Sha256Bytes", [64])
    ptau = z.ptau_toy(c.info.domain_log2 + 1, *TOX)
    path = tmp_path / "toy.ptau"
    path.write_bytes(ptau)
    base = z.Zkey.from_ptau(c, str(path))
    key = base.contribute(_le(S1))
    padded, plen = z.sha256_pad(b"ptau setup", 64)
    inputs = {"paddedIn": list(padded), "paddedInLength": plen}
    rs = _le(1234567) + _le(7654321)
    proofs = []
    for k in (key, z.Zkey.load(key.write(), circuit=c)):
        ctx = z.Context(c, k, device=0, max_batch=1)
        ctx.witness(c.pack_inputs(inputs), 1)
        proofs.append(ctx.prove(1, rs)[:2])
        ctx.close()
    assert proofs[0] == proofs[1]
    with pytest.raises(z.InsecureKeyError):
        z.register_circuit("ptau-base", c, base)
    z.register_circuit("ptau-key", c, key)
    out = z.generate_proof(inputs, "https://example.invalid/", "ptau-key")
    digest = hashlib.sha256(b"ptau setup").digest()
    assert out["publicSignals"] == [str((b >> (7 - j)) & 1) for b in digest for j in range(8)]
    assert z.verify_proof(out["proof"], out["publicSignals"], "https://example.invalid/", "ptau-key")


# ------------------------------------------------------------------------------------------------ EmailVerifier scale
def _resolver(key):
    return lambda n, t: [z.synthetic.key_record(key)]


def test_email_verifier_key_equals_the_seeded_toy_key():
    """EmailVerifier(640, 768), N = 2^21: a toy ptau from the seed's (tau, alpha, beta), then contribute(delta), gives the
    seeded toy key's A, B1, B2, L, H, alpha, beta and delta; its IC is gamma times the toy key's (gamma = 1 here)."""
    c = z.Circuit("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1])
    seed = 77
    buf = ctypes.create_string_buffer(160)
    assert L.zke_setup_toxic(seed, buf) == 0
    tau, alpha, beta, gamma, delta = (int.from_bytes(buf.raw[32 * i:32 * i + 32], "little") for i in range(5))
    ptau = z.ptau_toy(c.info.domain_log2 + 1, tau, alpha, beta)
    key = z.Zkey.from_ptau(c, ptau).contribute(_le(delta))
    del ptau
    toy = z.Zkey(c, seed=seed)
    got, want = product_sections(key), product_sections(toy)
    for name in ("A", "B1", "B2", "C", "H", "alpha1", "beta1", "delta1", "delta2"):
        assert got[name] == want[name], f"section {name} differs from the seeded toy key"
    ic_toy = [want["IC"][64 * i:64 * i + 64] for i in range(c.info.n_public + 1)]
    for i, p in enumerate(ic_toy):
        pt = (int.from_bytes(p[:32], "little"), int.from_bytes(p[32:], "little"))
        x, y = bn254.g1_mul(pt, gamma)
        assert got["IC"][64 * i:64 * i + 64] == _le(x) + _le(y), f"IC {i} is not gamma times the toy key's"
    del toy
    key_rs = (0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321)
    email = z.synthetic.make_signed_email(20, (k := z.synthetic.generate_key()), body_len=512)
    dk = z.verify_dkim_signature(email, resolver=_resolver(k))
    inputs = z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": 640, "maxBodyLength": 768})
    ctx = z.Context(c, key, device=0, max_batch=1)
    wt, status = ctx.witness(c.pack_inputs(inputs), 1)
    assert status == [-1]
    proofs, publics, _ = ctx.prove(1, _le(key_rs[0]) + _le(key_rs[1]))
    ctx.close()
    assert proofs == oracle_prove(c, got, wt, key_rs[0], key_rs[1], threads=16)
    proof, pubs = z.proof_to_json(proofs, publics, c.info.n_public)
    vk = key.vkey()
    assert z.verify(vk, pubs, proof) and bn254.groth16_verify(vk, pubs, proof)
    assert z.Verifier(vk).verify_batch([pubs], [proof]) == [True]
