"""Intra-proof sharding (DESIGN.md 6 (ii)) on ONE GPU: every rank of a 2-, 4- or 8-way proof in one process.

Each rank of zke_shard_begin / _mid / _end is one zke_ctx, and nothing ties a rank to its own device: G contexts opened
on device 0, with the two all-to-alls done as device copies between their vectors, run exactly the kernels G GPUs would
run - the row-mapped mat-vec, the cross-block NTT stages (log2 G = 1, 2, 3; Montgomery and fixed-operand twiddles), the
block-local transforms with the coset scale at the block's offset, the column quotient, the range and column
multi-exponentiations and the per-rank first-violated-row flag.  The driver below reuses the product's index views
(zkemail_b200.parallel.shard_views) and host combine, so those are checked too.  NCCL refuses two ranks on one device,
so the exchanges are plain copies with the semantics of dist.all_to_all.

References: the single-context proof at the same (r, s), the CPU oracle's proof, and per rank the oracle's partial points
of that rank's share (tests/test_shard_partials_host.py), so that a failure names the rank and the partial."""
import ctypes

import pytest

import zkemail_b200 as z
from zkemail_b200 import _lib as L
from zkemail_b200 import parallel
from oracle import bn254
from r1cs_gen import generate
from test_shard_partials_host import oracle_partials, row_owner
from zkutil import oracle_prove, product_sections, ref, ref_view

pytestmark = pytest.mark.gpu

RS = (0x2B1D0E5F6A7C8D9E0F1A2B3C4D5E6F708192A3B4C5D6E7F8, 0x7F6E5D4C3B2A19080F1E2D3C4B5A69788796A5B4C3D2E1F0)
PARTIAL_NAMES = (("A", 0, 64), ("B1", 64, 128), ("C", 128, 192), ("H", 192, 256), ("B2", 256, 384))


def _rs(k=0):
    return (RS[0] + k).to_bytes(32, "little") + (RS[1] + 3 * k).to_bytes(32, "little")


def _check(rc, err):
    if rc != 0:
        raise L.ZkeError(err.value.decode())


def shard_prove(ctxs, worlds=None):
    """One proof by the G = len(ctxs) contexts (all on device 0, one key, the same witness resident in each), as
    parallel.prove_sharded computes it on G GPUs.  worlds: the world size each rank is told (default G).
    Returns (the G 388-byte partials, the G public-signal byte strings)."""
    import torch
    G = len(ctxs)
    worlds = worlds or [G] * G
    err = ctypes.create_string_buffer(L.ERRCAP)
    for r, x in enumerate(ctxs):
        _check(L.zke_shard_begin(x.handle, r, worlds[r], err, L.ERRCAP), err)
    n = L.c_size_t()
    vecs = []
    for x in ctxs:
        vs = []
        for which in range(3):
            ptr = L.zke_shard_vector(x.handle, which, ctypes.byref(n))
            vs.append(torch.as_tensor(parallel._DevVec(ptr, n.value), device=torch.device("cuda", x.device)))
        vecs.append(vs)

    def exchange(to_rows):
        # dist.all_to_all(recv, send) on rank r: recv_r[g] <- send_g[r]; every send piece is read before any is written
        for which in range(3):
            views = [parallel.shard_views(vecs[r][which], r, G) for r in range(G)]
            send = [[t.clone() for t in (views[r][1] if to_rows else views[r][0])] for r in range(G)]
            for r in range(G):
                recv = views[r][0] if to_rows else views[r][1]
                for g in range(G):
                    recv[g].copy_(send[g][r])
        torch.cuda.synchronize()

    torch.cuda.synchronize()
    exchange(True)                                             # columns -> rows
    for x in ctxs:
        _check(L.zke_shard_mid(x.handle, err, L.ERRCAP), err)
    exchange(False)                                            # rows -> columns
    partials, publics = [], []
    for x in ctxs:
        part = ctypes.create_string_buffer(L.SHARD_PARTIAL_BYTES)
        pub = ctypes.create_string_buffer(max(1, 32 * x.n_public))
        _check(L.zke_shard_end(x.handle, part, pub, err, L.ERRCAP), err)
        partials.append(part.raw)
        publics.append(pub.raw[:32 * x.n_public])
    return partials, publics


def combine(zk, partials, rs):
    """zke_shard_combine: (return code, proof, status, error text)."""
    proof = ctypes.create_string_buffer(256)
    status = ctypes.c_int32(0)
    err = ctypes.create_string_buffer(L.ERRCAP)
    rc = L.zke_shard_combine(zk.handle, b"".join(partials), len(partials), rs, proof, ctypes.byref(status), err, L.ERRCAP)
    return rc, proof.raw, status.value, err.value.decode()


def open_ranks(c, zk, world):
    return [z.Context(c, zk, device=0, max_batch=1) for _ in range(world)]


def close_all(ctxs):
    for x in ctxs:
        x.close()


_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _release_cache():
    """Instances and keys are shared by the tests of this module and released after them."""
    yield
    _CACHE.clear()


def _instance(log_n):
    if ("instance", log_n) not in _CACHE:
        g = generate(log_n, seed=log_n)
        c = z.Circuit.from_r1cs(g["blob"])
        assert c.info.domain_log2 == log_n
        _CACHE["instance", log_n] = (g, c)
    return _CACHE["instance", log_n]


def _key(log_n):
    if ("key", log_n) not in _CACHE:
        _CACHE["key", log_n] = z.Zkey(_instance(log_n)[1], seed=300 + log_n)
    return _CACHE["key", log_n]


def _assert_partials(c, zk, partials, witness, world):
    """Each rank's partial points == the oracle's partials of that rank's share.  The point-range sums (A, B1, C, B2) of
    every rank are compared before any H: a wrong exchange spreads over the H scalars of every rank, so a failure in one
    rank's own work is named by its point-range sums."""
    sec = product_sections(zk)
    want = [oracle_partials(c, sec, witness, r, world, threads=16) for r in range(world)]
    for names in (("A", "B1", "C", "B2"), ("H",)):
        for r in range(world):
            for name, lo, hi in PARTIAL_NAMES:
                if name in names:
                    assert partials[r][lo:hi] == want[r][lo:hi], f"rank {r} of {world}: partial {name} differs from the oracle's"
    for r in range(world):
        assert partials[r][384:] == want[r][384:], f"rank {r} of {world}: a row is flagged"


# ------------------------------------------------------------------------------------------------ generated instances
# (G, log_n): smallest split at each G, and the larger blocks - at 2^17 / G = 4 the block transform is 2^15 (8+7 passes)
# and H uses c = 17 with the two-level sort; at 2^20 / G = 8 the block is 2^17 (6+6+5) and H uses c = 20
CASES = [(2, 12), (2, 13), (4, 14), (4, 17), (8, 16), (8, 20)]
PARTIAL_CASES = {(2, 12), (2, 13), (4, 14)}


def test_some_instance_splits_its_points_unevenly():
    """m % G != 0 somewhere: the point ranges [m r / G, m (r + 1) / G) then have unequal lengths."""
    uneven = [(G, k) for G, k in CASES if _instance(k)[1].info.n_vars % G]
    assert uneven, "every case splits its wires evenly"


# fixed-operand (Shoup) twiddles and coset factors, 64 bytes each, at the smallest 4- and 8-way splits
RUNS = [(G, k, False) for G, k in CASES] + [(4, 14, True), (8, 16, True)]


@pytest.mark.parametrize("world,log_n,shoup", RUNS, ids=[f"G{G}-2^{k}" + ("-shoup" if sh else "") for G, k, sh in RUNS])
def test_sharded_proof_equals_single_context_and_oracle(world, log_n, shoup, monkeypatch):
    monkeypatch.setenv("ZKE_NTT_SHOUP", "1" if shoup else "0")     # read when a context opens
    g, c = _instance(log_n)
    zk = _key(log_n)
    ctxs = open_ranks(c, zk, world)
    try:
        for x in ctxs:
            x.load_witness(g["witness"], 1)
        partials, publics = shard_prove(ctxs)
        proof, _, status = parallel.combine_partials(zk, b"".join(partials), world, _rs(), publics[0])
        assert status == -1
        want_pub = g["witness"][32:32 * (1 + c.info.n_public)]
        for r in range(world):
            assert publics[r] == want_pub, f"rank {r}: public signals differ from the witness's"
        single, single_pub, st = ctxs[0].prove(1, _rs())                    # an ordinary proof after a sharded one
        assert st == [-1] and single_pub == want_pub
        want = oracle_prove(c, product_sections(zk), g["witness"], RS[0], RS[1], threads=16)
        assert single == want, "single-context proof differs from the oracle's"
        if (world, log_n) in PARTIAL_CASES or proof != want:
            _assert_partials(c, zk, partials, g["witness"], world)
        assert proof == single, "sharded proof differs from the single-context proof"
        pj, pubs = z.proof_to_json(proof, publics[0], c.info.n_public)
        assert bn254.groth16_verify(zk.vkey(), pubs, pj)
    finally:
        close_all(ctxs)


def test_a_rank_told_the_wrong_world_is_named():
    """The checks above have teeth: rank 1 of 4 told it is one of 2 sums the wrong point range (and computes the wrong
    columns), so the combined proof is wrong and the per-rank comparison names rank 1."""
    world, log_n = 4, 14
    g, c = _instance(log_n)
    zk = _key(log_n)
    ctxs = open_ranks(c, zk, world)
    try:
        for x in ctxs:
            x.load_witness(g["witness"], 1)
        partials, publics = shard_prove(ctxs, worlds=[4, 2, 4, 4])
        rc, proof, status, _ = combine(zk, partials, _rs())
        assert (rc, status) == (0, -1)
        assert proof != oracle_prove(c, product_sections(zk), g["witness"], RS[0], RS[1], threads=16)
        with pytest.raises(AssertionError, match="rank 1 of 4: partial A differs"):
            _assert_partials(c, zk, partials, g["witness"], world)
    finally:
        close_all(ctxs)


def _witness_with(g, changes):
    """g's witness with the wires of `changes` (wire -> value) replaced."""
    w = bytearray(g["witness"])
    for wire, v in changes.items():
        w[32 * wire:32 * wire + 32] = v.to_bytes(32, "little")
    return bytes(w)


def _wire(g, wire):
    return int.from_bytes(g["witness"][32 * wire:32 * wire + 32], "little")


@pytest.mark.parametrize("world,log_n", [(4, 14), (8, 16)], ids=["G4-2^14", "G8-2^16"])
def test_bad_witness_names_the_lowest_violated_row_across_ranks(world, log_n):
    """Two violated quadratic rows checked by different ranks, the lower one not by rank 0: the combined status is the lower
    row, as the single-context prover and the oracle's check say, and the combine refuses to assemble a proof."""
    g, c = _instance(log_n)
    zk = _key(log_n)
    n = 1 << log_n
    quad = [(int(row), [int(w) for w in wires]) for row, wires in zip(g["quad_rows"], g["classes"]["quadratic"])]
    lo = next(q for q in quad if row_owner(q[0], n, world) not in (0,))
    hi = next(q for q in quad if q[0] > lo[0] and row_owner(q[0], n, world) not in (0, row_owner(lo[0], n, world)))
    # break x * y = z on both rows: z + 1
    bad = _witness_with(g, {q[1][2]: (_wire(g, q[1][2]) + 1) % z.FR_MODULUS for q in (lo, hi)})
    first = ref.zkref_check_r1cs(ctypes.byref(ref_view(c)), ctypes.create_string_buffer(bad, len(bad)))
    assert first == lo[0]
    ctxs = open_ranks(c, zk, world)
    try:
        for x in ctxs:
            x.load_witness(bad, 1)
        partials, publics = shard_prove(ctxs)
        flags = [int.from_bytes(p[384:388], "little") for p in partials]
        for r in range(world):
            want = lo[0] if r == row_owner(lo[0], n, world) else (hi[0] if r == row_owner(hi[0], n, world) else 0xFFFFFFFF)
            assert flags[r] == want, f"rank {r}: first violated row {flags[r]:#x}, expected {want:#x}"
        rc, proof, status, msg = combine(zk, partials, _rs())
        assert (rc, status, proof) == (1, lo[0], bytes(256)) and msg == f"Assert Failed: constraint {lo[0]}"
        with pytest.raises(z.AssertFailed):
            parallel.combine_partials(zk, b"".join(partials), world, _rs(), publics[0])
        _, _, single_status = ctxs[0].prove(1, _rs(), raise_on_fail=False)
        assert single_status == [lo[0]]
        # the same contexts prove a good witness afterwards
        for x in ctxs:
            x.load_witness(g["witness"], 1)
        partials, publics = shard_prove(ctxs)
        rc, proof, status, msg = combine(zk, partials, _rs())
        assert (rc, status) == (0, -1), msg
        assert proof == oracle_prove(c, product_sections(zk), g["witness"], RS[0], RS[1], threads=16)
    finally:
        close_all(ctxs)


def test_back_to_back_witnesses_leave_no_stale_state():
    """Two different witnesses proved one after the other on the same 8 contexts, then an ordinary proof on rank 0's
    context: each equals the single-context proof (on a context of its own) and the oracle's."""
    world, log_n = 8, 16
    g, c = _instance(log_n)
    zk = _key(log_n)
    # a second satisfying witness: every quadratic row's x + 1 with z = (x + 1) y, and the special values shifted
    changes = {}
    for x, y, zz in g["classes"]["quadratic"]:
        x1 = (_wire(g, int(x)) + 1) % z.FR_MODULUS
        changes[int(x)], changes[int(zz)] = x1, x1 * _wire(g, int(y)) % z.FR_MODULUS
    for w in g["classes"]["special"]:
        changes[int(w)] = (_wire(g, int(w)) + 12345) % z.FR_MODULUS
    w2 = _witness_with(g, changes)
    witnesses = [g["witness"], w2]
    sec = product_sections(zk)
    single = z.Context(c, zk, device=0, max_batch=1)
    ctxs = open_ranks(c, zk, world)
    try:
        want = []
        for k, w in enumerate(witnesses):
            single.load_witness(w, 1)
            p, _, st = single.prove(1, _rs(k))
            assert st == [-1] and p == oracle_prove(c, sec, w, RS[0] + k, RS[1] + 3 * k, threads=16)
            want.append(p)
        assert want[0] != want[1]
        for k, w in enumerate(witnesses):
            for x in ctxs:
                x.load_witness(w, 1)
            partials, publics = shard_prove(ctxs)
            proof, _, _ = parallel.combine_partials(zk, b"".join(partials), world, _rs(k), publics[0])
            assert proof == want[k], f"sharded proof of witness {k} differs from its single-context proof"
        p, _, _ = ctxs[0].prove(1, _rs(1))
        assert p == want[1], "ordinary proof after two sharded ones differs"
    finally:
        single.close()
        close_all(ctxs)


def test_refusals_leave_the_contexts_usable():
    g, c = _instance(12)
    zk = _key(12)
    err = ctypes.create_string_buffer(L.ERRCAP)

    def refused(rc, text):
        assert rc == -1 and text in err.value.decode(), err.value.decode()

    ctxs = open_ranks(c, zk, 2)
    no_key = z.Context(c, None, device=0, max_batch=1)
    no_witness = z.Context(c, zk, device=0, max_batch=1)
    try:
        refused(L.zke_shard_begin(ctxs[0].handle, 0, 2, err, L.ERRCAP), "no witness loaded")
        for x in ctxs:
            x.load_witness(g["witness"], 1)
        h = ctxs[0].handle
        refused(L.zke_shard_mid(h, err, L.ERRCAP), "zke_shard_mid out of order")
        part = ctypes.create_string_buffer(L.SHARD_PARTIAL_BYTES)
        refused(L.zke_shard_end(h, part, None, err, L.ERRCAP), "zke_shard_end out of order")
        for world in (0, 1, 3, 6, 16):
            refused(L.zke_shard_begin(h, 0, world, err, L.ERRCAP), "sharded proving supports 2, 4 or 8 GPUs")
        refused(L.zke_shard_begin(h, 2, 2, err, L.ERRCAP), "bad shard rank")
        refused(L.zke_shard_begin(h, -1, 2, err, L.ERRCAP), "bad shard rank")
        refused(L.zke_shard_begin(h, 0, 4, err, L.ERRCAP), "domain too small to shard")    # 2^12 < 2 * 2 + 10
        assert L.zke_shard_begin(h, 0, 2, err, L.ERRCAP) == 0
        refused(L.zke_shard_end(h, part, None, err, L.ERRCAP), "zke_shard_end out of order")
        refused(L.zke_shard_begin(no_key.handle, 0, 2, err, L.ERRCAP), "context was opened without a proving key")
        assert not L.zke_shard_vector(no_key.handle, 0, None)
        refused(L.zke_shard_begin(no_witness.handle, 0, 2, err, L.ERRCAP), "no witness loaded")
        # after all of that, the contexts prove
        partials, publics = shard_prove(ctxs)
        proof, _, status = parallel.combine_partials(zk, b"".join(partials), 2, _rs(), publics[0])
        assert status == -1 and proof == oracle_prove(c, product_sections(zk), g["witness"], RS[0], RS[1], threads=16)
    finally:
        close_all(ctxs + [no_key, no_witness])


def test_domain_too_small_for_eight_ranks():
    """2^15 < 2 * 3 + 10: eight ranks are refused, four (2^15 >= 14) are not."""
    g, c = _instance(15)
    zk = z.Zkey(c, seed=315)
    ctx = z.Context(c, zk, device=0, max_batch=1)
    err = ctypes.create_string_buffer(L.ERRCAP)
    try:
        ctx.load_witness(g["witness"], 1)
        assert L.zke_shard_begin(ctx.handle, 3, 8, err, L.ERRCAP) == -1
        assert "domain too small to shard" in err.value.decode()
        assert L.zke_shard_begin(ctx.handle, 3, 4, err, L.ERRCAP) == 0
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ a real circuit
@pytest.mark.parametrize("world", [2, 8])
def test_email_verifier_sharded_equals_single_context(world):
    """EmailVerifier(640, 768, 121, 17, 0, 0, 0, 0, 1), domain 2^21, with the witness made by the GPU witness kernel on
    every rank context as prove_sharded does."""
    c = z.Circuit("EmailVerifier", [640, 768, 121, 17, 0, 0, 0, 0, 1])
    assert c.info.domain_log2 == 21
    zk = _email_key(c)
    packed = _email_input(c)
    ctxs = open_ranks(c, zk, world)
    try:
        for x in ctxs:
            _, st = x.witness(packed, 1, want_witness=False)
            assert st == [-1]
        partials, publics = shard_prove(ctxs)
        proof, _, status = parallel.combine_partials(zk, b"".join(partials), world, _rs(5), publics[0])
        assert status == -1 and all(p == publics[0] for p in publics)
        single, single_pub, _ = ctxs[0].prove(1, _rs(5))
        assert single_pub == publics[0]
        assert proof == single, "sharded proof differs from the single-context proof"
        pj, pubs = z.proof_to_json(proof, publics[0], c.info.n_public)
        assert z.verify(zk.vkey(), pubs, pj)
    finally:
        close_all(ctxs)


def _email_key(c):
    if "email_key" not in _CACHE:
        _CACHE["email_key"] = z.Zkey(c, seed=31337)
    return _CACHE["email_key"]


def _email_input(c):
    if "email_input" not in _CACHE:
        key = z.synthetic.generate_key(seed=3)
        dk = z.verify_dkim_signature(z.synthetic.make_signed_email(77, key, body_len=512),
                                     resolver=lambda n_, t: [z.synthetic.key_record(key)])
        inputs = z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": 640, "maxBodyLength": 768})
        _CACHE["email_input"] = c.pack_inputs(inputs)
    return _CACHE["email_input"]
