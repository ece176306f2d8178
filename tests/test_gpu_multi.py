"""Multi-GPU (>= 2 devices, one process per GPU, NCCL) parity test of the sharded MSM with the fused NVLink
all-reduce of the partial commitments (csrc/peer.cu): sum over ranks == full MSM of the oracle.  Skipped on a
single-GPU machine (run `python -m pytest tests/test_gpu_multi.py -m gpu` on one with two or more)."""
import os
import socket
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import halo2_lib_b200 as h
    from oracle import oracle as orc, pyref
    from util import mont, rand_ints, witness_like_ints, affine_to_limbs
    ctx = h.Context(rank)
    stream = torch.cuda.Stream(device=rank)
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    h.connect_peers(ctx)
    k = 12
    n = 1 << k
    rng = np.random.default_rng(4242)  # same inputs on every rank
    g = affine_to_limbs([pyref.G1])[0]
    bases = ctx.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], pyref.R))
    cols = [mont(rand_ints(rng, n, pyref.R), pyref.R), mont(witness_like_ints(rng, n), pyref.R), mont(rand_ints(rng, n, pyref.R), pyref.R)]
    begin, count = h.shard_range(n, rank, world)
    params = h.ParamsKZG(ctx, k, g=bases, g_lagrange=bases, begin=begin, count=count)
    ok = True
    for it in range(3):  # several epochs through the same mailboxes
        d_cols = [torch.from_numpy(c[begin:begin + count].view(np.int64)).cuda() for c in cols]
        d_out = torch.zeros((3, 12), dtype=torch.int64, device="cuda")
        params.commit_batch_dev([0, 1, 0], [c.data_ptr() for c in d_cols], count, d_out.data_ptr())
        h.allreduce_points(ctx, d_out.data_ptr(), 3)
        ctx.synchronize()
        got = ctx.g1_normalize(d_out.cpu().numpy().view(np.uint64))
        for j in range(3):
            ok = ok and np.array_equal(got[j], orc.msm_pippenger(cols[j], bases, 2))
        cols = [np.roll(c, 1, axis=0) for c in cols]
    ret[rank] = bool(ok)
    dist.barrier()
    params.close()
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_msm_with_nvlink_allreduce():
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert dict(ret) == {r: True for r in range(world)}


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_single_process_device_group():
    """h2b_ctx_create_multi: ONE process drives all GPUs — the SRS is sharded inside h2b_srs_upload, h2b_msm_g1_batch returns
    the full sums (fused all-reduce over in-process peer mappings), the batched transforms are dealt round-robin"""
    import ctypes as C
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import halo2_lib_b200 as h
    from halo2_lib_b200._capi import lib
    from oracle import oracle as orc, pyref
    from util import mont, rand_ints, witness_like_ints, affine_to_limbs
    ndev = min(torch.cuda.device_count(), 4)
    grp = h.Context(list(range(ndev)))
    assert grp.device_count == ndev
    k = 12
    n = 1 << k
    rng = np.random.default_rng(515)
    g = affine_to_limbs([pyref.G1])[0]
    bases = grp.g1_fixed_base_mul(g, mont([3 + 5 * i for i in range(n)], pyref.R))
    bases_l = bases[::-1].copy()
    params = h.ParamsKZG(grp, k, g=bases, g_lagrange=bases_l)
    cols = [mont(rand_ints(rng, n, pyref.R), pyref.R), mont(witness_like_ints(rng, n), pyref.R), mont(rand_ints(rng, n, pyref.R), pyref.R),
            mont(witness_like_ints(rng, n), pyref.R), np.zeros((n, 4), dtype=np.uint64)]
    for rep in range(3):  # several epochs through the same mailboxes
        outs = params.commit_batch([0, 1, 0, 1, 0], cols)
        for j, (b, c) in enumerate(zip([0, 1, 0, 1, 0], cols)):
            assert np.array_equal(grp.g1_normalize(outs[j].reshape(1, 12))[0], orc.msm_pippenger(c, bases if b == 0 else bases_l, 2)), (rep, j)
        assert np.array_equal(grp.g1_normalize(params.commit(cols[0]).reshape(1, 12))[0], orc.msm_pippenger(cols[0], bases, 2))
        cols = [np.roll(c, 1, axis=0) for c in cols]
    dom = h.EvaluationDomain(grp, 5, k)
    polys = [mont(rand_ints(rng, n, pyref.R), pyref.R) for _ in range(7)]
    got = dom.lagrange_to_coeff_many(polys)
    for p, q in zip(polys, got):
        assert np.array_equal(q, orc.lagrange_to_coeff(p, k))
    cf, ex = dom.lagrange_to_coeff_and_extended_many(polys[:5])
    for p, c, e in zip(polys, cf, ex):
        assert np.array_equal(c, orc.lagrange_to_coeff(p, k))
        assert np.array_equal(e, orc.coeff_to_extended(c, dom.extended_k))
    params.close()
    grp.close()
