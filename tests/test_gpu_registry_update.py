"""In-place registry updates on the GPU (zke_registry_*, KeyRegistry.update / append).  After every call of seeded random
update sequences - single and batched replacements, revocations to 0, appends and calls mixing both - the resident
levels equal zke_merkle_build over the resulting leaves byte for byte, and oracle/merkle.levels where the Python oracle
is affordable; the patched KeyRegistry.levels equal both, and KeyRegistry.path equals the path gathered by
zke_registry_nodes and oracle/merkle.path.  Refused updates leave the resident tree unchanged, growth across several
capacity doublings keeps every level, and an app proves against a registry after a revocation and an append."""
import ctypes
import functools
import random

import pytest

import zkemail_b200 as z
from oracle import merkle
from test_app_commit import SALT, commit_body, commit_spec
from test_domain_registry import domain_spec
from zkemail_b200.registry import _split_levels

pytestmark = pytest.mark.gpu

R = z.FR_MODULUS
L = z._lib


def _flat(levels):
    return b"".join(x.to_bytes(32, "little") for lvl in levels for x in lvl)


def _resident(reg):
    """zke_registry_levels of the registry's resident tree."""
    h, err = reg._handle(), ctypes.create_string_buffer(L.ERRCAP)
    need = L.zke_registry_levels(h, None, 0, err, L.ERRCAP)
    assert need > 0, err.value
    buf = ctypes.create_string_buffer(need)
    assert L.zke_registry_levels(h, buf, need, err, L.ERRCAP) == need, err.value
    assert L.zke_registry_levels(h, buf, need - 1, err, L.ERRCAP) == -2
    return buf.raw


def _built(leaves, depth):
    err = ctypes.create_string_buffer(L.ERRCAP)
    data = b"".join(x.to_bytes(32, "little") for x in leaves)
    need = L.zke_merkle_build(data, len(leaves), depth, 0, None, 0, err, L.ERRCAP)
    buf = ctypes.create_string_buffer(need)
    assert L.zke_merkle_build(data, len(leaves), depth, 0, buf, need, err, L.ERRCAP) == need, err.value
    return buf.raw


def _gathered_path(reg, i):
    d = reg.depth
    lv, ix = (ctypes.c_uint32 * d)(*range(d)), (ctypes.c_uint64 * d)(*((i >> l) ^ 1 for l in range(d)))
    out, err = ctypes.create_string_buffer(32 * d), ctypes.create_string_buffer(L.ERRCAP)
    assert L.zke_registry_nodes(reg._handle(), lv, ix, d, out, err, L.ERRCAP) == 0, err.value
    return [int.from_bytes(out.raw[32 * l:32 * l + 32], "little") for l in range(d)]


def _check(reg, want, oracle, touched=()):
    """The invariant after one call; `want` is the leaf list kept independently of the registry."""
    assert reg.leaves == want
    assert L.zke_registry_count(reg._handle()) == len(want)
    raw = _resident(reg)
    assert raw == _built(want, reg.depth), "resident levels differ from a from-scratch build"
    assert _flat(reg.levels) == raw, "patched KeyRegistry.levels differ from the resident levels"
    lv = merkle.levels(want, reg.depth) if oracle else _split_levels(raw, len(want), reg.depth)
    if oracle:
        assert reg.levels == lv, "levels differ from the oracle"
    rng = random.Random(len(want))
    for i in sorted({0, len(want) - 1, rng.randrange(len(want))} | set(list(touched)[:2])):
        idx, sib = reg.path(i)
        assert idx == i and sib == _gathered_path(reg, i) == merkle.path(lv, i), i
    if oracle:
        assert merkle.check_path(reg.root, want[-1], len(want) - 1, reg.path(len(want) - 1)[1])


def _step(rng, reg, want, max_batch):
    """One random call: a single or batched replacement, revocations, an append, or replacements mixed with appends.
    Returns the touched indices."""
    count, room = len(want), (1 << reg.depth) - len(want)
    kind = rng.choice(["single", "batch", "revoke", "append", "mixed"])
    if kind == "append" and room:
        leaves = [rng.randrange(R) for _ in range(rng.randint(1, min(room, max_batch)))]
        assert reg.append(leaves) == list(range(count, count + len(leaves)))
        want.extend(leaves)
        return range(count, count + len(leaves))
    if kind == "single":
        changes = {rng.randrange(count): rng.randrange(R)}
    elif kind == "revoke":
        idx = {count - 1} | set(rng.sample(range(count), min(count, rng.randint(1, 8))))
        changes = {i: 0 for i in idx}
    else:
        changes = {i: rng.randrange(R) for i in rng.sample(range(count), min(count, rng.randint(2, max_batch)))}
    pairs = list(changes.items())
    if kind == "mixed" and room:
        a = rng.randint(1, min(room, max_batch))
        pairs += [(count + j, rng.randrange(R)) for j in range(a)]
    rng.shuffle(pairs)
    reg.update(pairs)
    for i, x in pairs:
        if i < len(want):
            want[i] = x
    want.extend(x for i, x in sorted(p for p in pairs if p[0] >= count))
    return [i for i, _ in pairs]


@pytest.mark.parametrize("depth,count,steps,max_batch,oracle", [
    (1, 1, 8, 2, True),
    (4, 3, 12, 6, True),
    (10, 1000, 8, 600, True),
    (20, (1 << 16) + 3, 8, 3000, False),
    (32, 5, 8, 4, True),
], ids=["depth1", "depth4", "depth10", "depth20", "depth32"])
def test_random_update_sequences(depth, count, steps, max_batch, oracle):
    rng = random.Random(depth)
    want = [rng.randrange(R) for _ in range(count)]
    reg = z.KeyRegistry.from_leaves(want, depth)
    want = list(want)
    _check(reg, want, oracle)
    for _ in range(steps):
        _check(reg, want, oracle, _step(rng, reg, want, max_batch))
    if depth <= 10:                                   # fill the tree, then a call that replaces every leaf
        if len(want) < 1 << depth:
            new = [rng.randrange(R) for _ in range((1 << depth) - len(want))]
            reg.update({len(want) + j: x for j, x in enumerate(new)} | {0: 0})
            want[0] = 0
            want.extend(new)
            _check(reg, want, oracle)
        everything = {i: rng.randrange(R) for i in range(len(want))}
        reg.update(everything)
        want = [everything[i] for i in range(len(want))]
        _check(reg, want, oracle)
        assert reg.root == merkle.root(want, depth)
    assert L.zke_registry_device_ms() > 0
    reg.close()
    reg.update({0: 7})                                # a closed registry reopens from its levels
    want[0] = 7
    _check(reg, want, oracle)
    reg.close()


def test_refused_updates_leave_the_tree_unchanged():
    """zke_registry_update refuses each bad update itself, with KeyRegistry.update's message, before any device write."""
    rng = random.Random(3)
    reg = z.KeyRegistry.from_leaves([rng.randrange(R) for _ in range(1020)], 10)
    before = _resident(reg)
    err = ctypes.create_string_buffer(L.ERRCAP)
    for pairs in ([(7, 1), (1020, 2), (7, 3)], [(1020, 1), (1022, 2)], [(1020 + j, j) for j in range(5)],
                  [(0, 1), (1020, R), (3, 3)], [(5, 1), (1024, 1)]):
        with pytest.raises(ValueError) as e:
            reg.update(pairs)
        idx = (ctypes.c_uint64 * len(pairs))(*(i for i, _ in pairs))
        data = b"".join(x.to_bytes(32, "little") for _, x in pairs)
        assert L.zke_registry_update(reg._handle(), idx, data, len(pairs), err, L.ERRCAP) < 0
        assert err.value.decode() == str(e.value)
        assert _resident(reg) == before and L.zke_registry_count(reg._handle()) == 1020
    assert L.zke_registry_update(reg._handle(), None, None, 0, err, L.ERRCAP) == 0
    lv, ix, out = (ctypes.c_uint32 * 1)(11), (ctypes.c_uint64 * 1)(0), ctypes.create_string_buffer(32)
    assert L.zke_registry_nodes(reg._handle(), lv, ix, 1, out, err, L.ERRCAP) < 0 and b"above the root" in err.value
    lv[0], ix[0] = 2, 256
    assert L.zke_registry_nodes(reg._handle(), lv, ix, 1, out, err, L.ERRCAP) < 0 and b"index 256 is outside level 2" in err.value
    ix[0] = 255                                       # past the 255 nodes of level 2, inside the tree: zeros[2]
    assert L.zke_registry_nodes(reg._handle(), lv, ix, 1, out, err, L.ERRCAP) == 0
    assert int.from_bytes(out.raw, "little") == merkle.zeros(10)[2]
    assert _resident(reg) == before
    reg.close()


def test_capacity_growth_keeps_every_level():
    """One leaf, then appends of 1, 2, 4, ... leaves: the capacity doubles nine times, to the full tree of depth 9."""
    rng = random.Random(4)
    want = [rng.randrange(R)]
    reg = z.KeyRegistry.from_leaves(want, 9)
    for a in (1, 2, 4, 8, 16, 32, 64, 128, 3, 253):
        leaves = [rng.randrange(R) for _ in range(a)]
        reg.append(leaves)
        want += leaves
        assert _resident(reg) == _built(want, 9)
        assert _flat(reg.levels) == _resident(reg)
    assert len(want) == 512 and reg.levels == merkle.levels(want, 9)
    reg.close()


# ---- the app -----------------------------------------------------------------------------------------------------------

DEPTH = 10
_key = functools.lru_cache(maxsize=None)(lambda seed: z.synthetic.generate_key(seed=seed))


def _signed(i, domain, seed):
    key = _key(seed)
    em = z.synthetic.make_signed_email(i, key, domain=domain, body_override=commit_body(str(1000 + i), "a note"))
    return z.verify_dkim_signature(em, resolver=lambda n, t: [z.synthetic.key_record(key)])


def _prove(spec, c, inputs, seed):
    from oracle import bn254
    zk = z.Zkey(c, seed=seed)
    ctx = z.Context(c, zk, device=0, max_batch=1)
    _, status = ctx.witness(c.pack_inputs(inputs), 1, want_witness=False)
    assert status == [-1]
    proofs, publics, _ = ctx.prove(1)
    proof, pubs = z.proof_to_json(proofs, publics, c.info.n_public)
    assert z.verify(zk.vkey(), pubs, proof) and bn254.groth16_verify(zk.vkey(), pubs, proof)
    return z.decode_app_outputs(spec, pubs)


@pytest.mark.parametrize("bound", [False, True], ids=["pubkeyHash", "domainKey"])
def test_revoke_then_append_the_signer(bound):
    """A 1,000-key registry holding the signer at slot 333: revoking its leaf makes generate_app_inputs refuse the
    email; appending the signer's leaf at index 1,000 lets it prove again, publishing the updated root."""
    seed, slot, domain = 81, 333, "corp81.com"
    rng = random.Random(10)
    key = z.synthetic.key_record(_key(seed))
    if bound:
        spec = domain_spec(1, "dkim", depth=DEPTH)
        pairs = [(f"filler{i}.example", rng.getrandbits(2048) | (1 << 2047) | 1) for i in range(1000)]
        pairs[slot] = (domain, key)
        reg = z.KeyRegistry.build_domains(pairs, DEPTH)
        leaf = z.registry.domain_key_leaves([(domain, key)])[0]
        refusal = f'not registered for domain "{domain}"'
    else:
        spec = dict(commit_spec(1), keyRegistryDepth=DEPTH)
        keys = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(1000)]
        keys[slot] = key
        reg = z.KeyRegistry.build(keys, DEPTH)
        leaf = z.registry.pubkey_hashes([key])[0]
        refusal = "not in the registry"
    assert reg.leaves[slot] == leaf
    c = z.Circuit.from_spec(spec)
    dk = _signed(7, domain, seed)
    externals = {"senderSalt": SALT, "recipient": 1}
    old_root = reg.root

    reg.update({slot: 0})
    assert reg.root != old_root
    with pytest.raises(ValueError, match=refusal):
        z.generate_app_inputs(dk, spec, externals, params={"registry": reg})

    assert reg.append([leaf]) == [1000]
    inputs = z.generate_app_inputs(dk, spec, externals, params={"registry": reg})
    assert inputs["registryIndex"] == "1000"
    scratch = z.KeyRegistry.from_leaves(reg.leaves, DEPTH, domain_bound=bound)
    assert scratch.levels == reg.levels
    out = _prove(spec, c, inputs, seed=31 + bound)
    assert out["registryRoot"] == reg.root == scratch.root == merkle.root(reg.leaves, DEPTH)
    assert out["registryRoot"] != old_root
    if bound:
        assert out["dkimDomain"] == domain
    reg.close()
