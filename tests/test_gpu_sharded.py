"""Intra-proof sharding on real GPUs (SURVEY 8(e)(ii)): ONE proof computed by 2 (or 4 / 8) GPUs together - mat-vec and
NTTs split 4-step style with two NCCL all-to-alls, every multi-exponentiation sharded over the points, partial sums
all-gathered - must be bit-identical to the single-GPU proof at the same (r, s).  Needs `world` visible GPUs (skipped
otherwise).  tests/test_gpu_shard_one_device.py runs the same device code for 2, 4 and 8 ranks on one GPU."""
import os
import socket
import sys

import pytest

pytestmark = pytest.mark.gpu

CIRCUIT = os.environ.get("SHARD_TEST_CIRCUIT", "EmailVerifier:640,768,121,17,0,0,0,0,1")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "zk-email-verify_b200", "host"), os.path.join(root, "tests")):
        sys.path.insert(0, p)
    import time
    import torch
    import torch.distributed as dist
    import zkemail_b200 as z
    from zkemail_b200.parallel import prove_sharded
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    name, _, params = CIRCUIT.partition(":")
    params = [int(x) for x in params.split(",")]
    c = z.Circuit(name, params)
    zk = z.Zkey(c, seed=31337, device=rank)            # the same (seeded) key on every GPU
    ctx = z.Context(c, zk, device=rank, max_batch=1)
    # every rank must prove the same email: rank 0 makes it (RSA keys are not seedable) and broadcasts it
    blob = [None, None]
    if rank == 0:
        rsa_key = z.synthetic.generate_key()
        blob = [z.synthetic.make_signed_email(77, rsa_key, body_len=min(512, params[1] - 128)), z.synthetic.key_record(rsa_key)]
    dist.broadcast_object_list(blob, src=0)
    dk = z.verify_dkim_signature(blob[0], resolver=lambda n, t: [blob[1]])
    inputs = z.generate_email_verifier_inputs_from_dkim_result(dk, {"maxHeadersLength": params[0], "maxBodyLength": params[1]})
    packed = c.pack_inputs(inputs)
    rs = (0x1357924680ACE).to_bytes(32, "little") + (0x2468ACE013579).to_bytes(32, "little")
    prove_sharded(ctx, packed, rs)                       # warm-up (NCCL communicators, allocations)
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    proof, publics, status = prove_sharded(ctx, packed, rs)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    single = None
    if rank == 0:
        ctx.witness(packed, 1, want_witness=False)
        t1 = time.perf_counter()
        ctx.witness(packed, 1, want_witness=False)
        single, single_pub, _ = ctx.prove(1, rs)
        dt_single = time.perf_counter() - t1
        pj, pubs = z.proof_to_json(proof, publics, c.info.n_public)
        q.put((rank, proof == single, publics == single_pub, status, z.verify(zk.vkey(), pubs, pj), dt, dt_single, c.info.domain_log2))
    else:
        q.put((rank, True, True, status, True, dt, 0.0, c.info.domain_log2))
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_proof_is_bit_identical_to_single_gpu(world):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted(q.get(timeout=1500) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    rank0 = results[0]
    assert rank0[1] and rank0[2], "sharded proof differs from the single-GPU proof"
    assert rank0[3] == -1 and rank0[4]
    print("sharded proof across %d GPUs (domain 2^%d): %.1f ms; single GPU witness + prove: %.1f ms" % (world, rank0[7], 1e3 * rank0[5], 1e3 * rank0[6]))
