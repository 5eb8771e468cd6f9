"""world_size-2 gloo test of the multi-GPU host logic (proof-level sharding + ordered gather); no GPU involved."""
import os
import socket
import sys

import torch.multiprocessing as mp


def _worker(rank, world, port, n_items, n_public, q):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zk-email-verify_b200", "host"))
    import torch.distributed as dist
    from zkemail_b200.parallel import shard_range, gather_proofs
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mine = shard_range(n_items, rank, world)
    proofs = b"".join(bytes([i % 251]) * 256 for i in mine)                 # stand-ins for this shard's proofs
    publics = b"".join(bytes([(i * 7) % 253]) * (32 * n_public) for i in mine)
    all_proofs, all_publics = gather_proofs(proofs, publics, n_items, n_public)
    q.put((rank, list(mine), all_proofs, all_publics))
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_shard_range_partitions():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zk-email-verify_b200", "host"))
    from zkemail_b200.parallel import shard_range
    for n in (0, 1, 7, 64, 1000):
        for world in (1, 2, 3, 8):
            cover = [i for r in range(world) for i in shard_range(n, r, world)]
            assert cover == list(range(n))
            sizes = [len(shard_range(n, r, world)) for r in range(world)]
            assert max(sizes) - min(sizes) <= 1


def test_two_rank_gather_is_ordered_and_complete():
    world, n_items, n_public = 2, 7, 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n_items, n_public, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    expect_proofs = b"".join(bytes([i % 251]) * 256 for i in range(n_items))
    expect_publics = b"".join(bytes([(i * 7) % 253]) * (32 * n_public) for i in range(n_items))
    shards = sorted(r[1] for r in results)
    assert shards == [[0, 1, 2, 3], [4, 5, 6]]
    for _, _, proofs, publics in results:
        assert proofs == expect_proofs and publics == expect_publics


# ---------------------------------------------------------------------------------------------------------------------
# Intra-proof sharding (SURVEY 8(e)(ii)): the two pieces of host logic of zkemail_b200.parallel.prove_sharded that do
# not need a GPU - the all-to-all index logic of the NTT exchanges and the all-gather + combine of the partial points -
# on world_size 2 over gloo.
def _exchange_worker(rank, world, port, q):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "zk-email-verify_b200", "host"))
    import torch
    import torch.distributed as dist
    from zkemail_b200.parallel import shard_exchange
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    n = 8 * world * world
    m, c = n // world, n // (world * world)
    # column layout: this rank holds (block g, its columns) for every g; everything else is poison
    vec = torch.full((n, 4), -1, dtype=torch.int64)
    for g in range(world):
        for j in range(rank * c, (rank + 1) * c):
            vec[g * m + j] = g * m + j
    shard_exchange(vec, rank, world, True)
    row_ok = bool((vec[rank * m:(rank + 1) * m, 0] == torch.arange(rank * m, (rank + 1) * m)).all())
    vec[rank * m:(rank + 1) * m] *= 3                      # "block-local work" on the row block
    poison = torch.ones(n, dtype=torch.bool)
    poison[rank * m:(rank + 1) * m] = False
    vec[poison] = -7
    shard_exchange(vec, rank, world, False)
    col_ok = all(int(vec[g * m + j, 0]) == 3 * (g * m + j) for g in range(world) for j in range(rank * c, (rank + 1) * c))
    q.put((rank, row_ok, col_ok))
    dist.destroy_process_group()


def test_shard_exchange_moves_columns_to_rows_and_back():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_exchange_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert sorted(results) == [(0, True, True), (1, True, True)]


def _combine_worker(rank, world, port, q):
    """Each rank sums its share of the five multi-exponentiations with the Python oracle's curve arithmetic (the shares of
    the engine's column layout, tests/test_shard_partials_host.py), the partial points are all-gathered over gloo and combined by the product's host routine (zke_shard_combine_raw)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "zk-email-verify_b200", "host"), os.path.join(root, "tests")):
        sys.path.insert(0, p)
    import ctypes
    import torch
    import torch.distributed as dist
    import zkemail_b200 as z
    from zkemail_b200 import _lib as L
    from zkemail_b200 import iden3_binfile as B
    from test_shard_partials_host import column_positions, point_range
    from zkutil import oracle_setup, oracle_prove, oracle_witness
    from oracle import bn254
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    P = z.FR_MODULUS
    c = z.Circuit("FpMul", [2, 4])
    info = c.info
    n, m, l = 1 << info.domain_log2, info.n_vars, info.n_public
    toxic = (1234567, 11, 22, 33, 44)
    sec = oracle_setup(c, toxic)
    w = oracle_witness(c, {"a": [1, 0, 1, 0], "b": [0, 1, 1, 0], "p": [1, 1, 1, 1]})
    vals = [w[i] for i in range(m)]
    r, s = 987654321, 123456789
    want = oracle_prove(c, sec, w.raw(), r, s, threads=1)
    # scalars of the H multi-exponentiation: a o b - c on the coset (SURVEY A.7), by direct O(N^2) evaluation
    r1 = B.read_r1cs(B.write_r1cs(c))
    ev = lambda lc: sum(v * vals[k] for k, v in lc.items()) % P
    a = [ev(row[0]) for row in r1["constraints"]] + [vals[j] for j in range(l + 1)]
    b = [ev(row[1]) for row in r1["constraints"]] + [0] * (l + 1)
    a += [0] * (n - len(a)); b += [0] * (n - len(b))
    cc = [x * y % P for x, y in zip(a, b)]
    omega = pow(5, (P - 1) // n, P)
    g = pow(5, (P - 1) // (2 * n), P)
    def coset_evals(ev_on_domain):
        n_inv = pow(n, -1, P)
        coef = [sum(ev_on_domain[i] * pow(omega, -i * k, P) for i in range(n)) * n_inv % P for k in range(n)]
        return [sum(coef[k] * pow(g * pow(omega, i, P), k, P) for k in range(n)) % P for i in range(n)]
    a2, b2, c2 = coset_evals(a), coset_evals(b), coset_evals(cc)
    d = [(x * y - zc) % P for x, y, zc in zip(a2, b2, c2)]
    g1pt = lambda raw: None if raw == bytes(64) else (int.from_bytes(raw[:32], "little"), int.from_bytes(raw[32:], "little"))
    g2pt = lambda raw: None if raw == bytes(128) else ((int.from_bytes(raw[:32], "little"), int.from_bytes(raw[32:64], "little")),
                                                       (int.from_bytes(raw[64:96], "little"), int.from_bytes(raw[96:], "little")))
    def msm1(section, scalars, idx):
        acc = None
        for i in idx:
            p = g1pt(sec[section][64 * i:64 * i + 64])
            if p is not None and scalars[i]:
                acc = bn254.g1_add(acc, bn254.g1_mul(p, scalars[i]))
        return acc
    # the engine's shares (zke_shard_end): a contiguous point range, and for H the rank's columns of every block
    mine_pts, mine_h = point_range(m, rank, world), [int(i) for i in column_positions(n, rank, world)]
    pa, pb1, pc, ph = msm1("A", vals, mine_pts), msm1("B1", vals, mine_pts), msm1("C", vals, mine_pts), msm1("H", d, mine_h)
    pb2 = None
    for i in mine_pts:
        p = g2pt(sec["B2"][128 * i:128 * i + 128])
        if p is not None and vals[i]:
            pb2 = bn254.g2_add(pb2, bn254.g2_mul(p, vals[i]))
    le = lambda v: int(v).to_bytes(32, "little")
    enc1 = lambda p: bytes(64) if p is None else le(p[0]) + le(p[1])
    enc2 = lambda p: bytes(128) if p is None else le(p[0][0]) + le(p[0][1]) + le(p[1][0]) + le(p[1][1])
    block = enc1(pa) + enc1(pb1) + enc1(pc) + enc1(ph) + enc2(pb2) + (0xffffffff).to_bytes(4, "little")
    assert len(block) == L.SHARD_PARTIAL_BYTES
    mine = torch.frombuffer(bytearray(block), dtype=torch.uint8)
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    allp = b"".join(bytes(t.numpy()) for t in gathered)
    key_points = sec["alpha1"] + sec["beta1"] + sec["delta1"] + sec["beta2"] + sec["delta2"]
    proof = ctypes.create_string_buffer(256)
    status = ctypes.c_int32(0)
    err = ctypes.create_string_buffer(512)
    rs = le(r) + le(s)
    rc = L.zke_shard_combine_raw(key_points, allp, world, rs, proof, ctypes.byref(status), err, 512)
    # a rank that saw a violated row makes the combined result an "Assert Failed"
    bad = bytearray(allp)
    bad[384:388] = (17).to_bytes(4, "little")
    st2 = ctypes.c_int32(0)
    rc_bad = L.zke_shard_combine_raw(key_points, bytes(bad), world, rs, ctypes.create_string_buffer(256), ctypes.byref(st2), err, 512)
    q.put((rank, rc, status.value, proof.raw == want, rc_bad, st2.value, err.value.decode()))
    dist.destroy_process_group()


def test_two_rank_partial_points_combine_to_the_oracle_proof():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_combine_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, rc, status, same, rc_bad, st_bad, msg in results:
        assert rc == 0 and status == -1 and same, "combined proof differs from the unsharded oracle proof"
        assert rc_bad == 1 and st_bad == 17 and "Assert Failed" in msg
