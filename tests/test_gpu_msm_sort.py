"""The MSM bucket sort (coarse bins, then the buckets inside each bin) on the shapes that stress it: one bucket holding every
entry, digits only in the first and the last coarse bin, 16-MSM groups over two tables, ad-hoc bases at their largest window,
shards that are not powers of two, and the k = 19 grouping of a prover phase.  Commitments are compared with the CPU oracle or
with the closed form sum_i s_i a_i * G for bases a_i * G."""
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *

pytestmark = pytest.mark.gpu
R = pyref.R


@pytest.fixture(scope="module")
def h2b():
    import halo2_lib_b200 as h
    return h


@pytest.fixture(scope="module")
def ctx(h2b):
    c = h2b.Context(0)
    yield c
    c.close()


def norm(ctx, xyz):
    return ctx.g1_normalize(np.asarray(xyz, dtype=np.uint64).reshape(1, 12))[0]


def bases(ctx, n, a0, delta):
    """b_i = (a0 + i*delta) * G, built on the GPU"""
    return ctx.g1_fixed_base_mul(affine_to_limbs([pyref.G1])[0], mont([a0 + i * delta for i in range(n)], R))


def closed_form(sc, a0, delta):
    return pyref.g1_mul(sum(s * (a0 + i * delta) for i, s in enumerate(sc)) % R, pyref.G1)


def affine(ctx, xyz):
    return jac_limbs_to_affine(norm(ctx, xyz))


def test_sort_one_bucket_holds_every_entry(ctx, h2b):
    """a column of ones at 2^20: every entry is digit 1 of window 0, so one bucket and one coarse bin hold everything"""
    k = 20
    n = 1 << k
    a0, delta = 17, 29
    B = bases(ctx, n, a0, delta)
    S = np.repeat(mont([1], R), n, axis=0)
    params = h2b.ParamsKZG(ctx, k, g=B)
    try:
        got = affine(ctx, params.commit(S))
    finally:
        params.close()
    assert got == pyref.g1_mul((a0 * n + delta * n * (n - 1) // 2) % R, pyref.G1)


def test_sort_first_and_last_coarse_bin(ctx, h2b):
    """k = 16 (c = 16, 16 windows, 2^15 buckets): every digit is in [1, 128] or [2^15 - 127, 2^15], i.e. in the first or the
    last coarse bin; the top window takes small digits so that the scalar stays below r"""
    k, c, W = 16, 16, 16
    n = 1 << k
    rng = np.random.default_rng(16)
    half = 1 << (c - 1)
    lo = rng.integers(1, 129, size=(n, W))
    hi = rng.integers(half - 127, half + 1, size=(n, W))
    pick = rng.random((n, W)) < 0.5
    pick[:, W - 1] = True
    dig = np.where(pick, lo, hi)
    sc = [sum(int(dig[i, w]) << (c * w) for w in range(W)) for i in range(n)]
    assert max(sc) < R
    a0, delta = 5, 11
    B = bases(ctx, n, a0, delta)
    params = h2b.ParamsKZG(ctx, k, g=B)
    try:
        got = affine(ctx, params.commit(mont(sc, R)))
    finally:
        params.close()
    assert got == closed_form(sc, a0, delta)


@pytest.mark.parametrize("group", [16, 2])
def test_sort_group_of_16_two_tables(h2b, group):
    """16 MSMs over two tables: zero, one-hot, witness-like and uniform columns; one pipeline of 16 and eight groups of two
    (more groups than lanes: the host-pointer call refills a lane's staging buffer once the sort of the lane's previous group
    has read it)"""
    import torch
    c = h2b.Context(0)
    c.set_option("msm.batch_group", group)
    try:
        k, m = 12, 16
        n = 1 << k
        rng = np.random.default_rng(1600 + group)
        Bm = bases(c, n, 3, 5)
        Bl = bases(c, n, 1001, 7)
        cols = []
        for j in range(m):
            if j % 4 == 0:
                sc = [0] * n
            elif j % 4 == 1:
                sc = [0] * n
                sc[(j * 97) % n] = rand_ints(rng, 1, R)[0]
            elif j % 4 == 2:
                sc = witness_like_ints(rng, n)
            else:
                sc = rand_ints(rng, n, R)
            cols.append(mont(sc, R))
        basis = [(j // 2) % 2 for j in range(m)]
        want = [orc.msm_pippenger(cols[j], Bl if basis[j] else Bm) for j in range(m)]
        params = h2b.ParamsKZG(c, k, g=Bm, g_lagrange=Bl)
        try:
            outs = params.commit_batch(basis, cols)  # host pointers
            for j in range(m):
                assert np.array_equal(norm(c, outs[j]), want[j]), (j, "host")
            d_cols = [torch.from_numpy(x.view(np.int64)).cuda() for x in cols]
            d_out = torch.zeros((m, 12), dtype=torch.int64, device="cuda")
            params.commit_batch_dev(basis, [t.data_ptr() for t in d_cols], n, d_out.data_ptr())
            torch.cuda.synchronize()
            outs = d_out.cpu().numpy().view(np.uint64)
            for j in range(m):
                assert np.array_equal(norm(c, outs[j]), want[j]), (j, "dev")
        finally:
            params.close()
    finally:
        c.close()


def test_sort_adhoc_largest_window(ctx, h2b):
    """ad-hoc bases use c = 16 from n > 2^19: 16 bucket sets of 2^15 buckets; n is not a power of two"""
    n = (1 << 19) + 3
    rng = np.random.default_rng(19)
    a0, delta = 7, 3
    B = bases(ctx, n, a0, delta)
    sc = rand_ints(rng, n // 2, R) + witness_like_ints(rng, n - n // 2)
    got = affine(ctx, h2b.best_multiexp(ctx, mont(sc, R), B))
    assert got == closed_form(sc, a0, delta)


def test_sort_odd_shard(ctx, h2b):
    k = 14
    n = 1 << k
    begin, count = 1234, 9999
    rng = np.random.default_rng(14)
    B = bases(ctx, n, 2, 9)
    cols = [mont(rand_ints(rng, count, R), R), mont(witness_like_ints(rng, count), R)]
    p = h2b.ParamsKZG(ctx, k, g=B, begin=begin, count=count)
    try:
        outs = p.commit_batch([0, 0], cols)
        for j in range(2):
            assert np.array_equal(norm(ctx, outs[j]), orc.msm_pippenger(cols[j], B[begin:begin + count])), j
    finally:
        p.close()


@pytest.fixture(scope="module")
def k19_columns():
    rng = np.random.default_rng(1919)
    n = 1 << 19
    kinds = ["uniform", "witness", "uniform", "zero", "witness", "uniform"]
    sc = [rand_ints(rng, n, R) if t == "uniform" else witness_like_ints(rng, n) if t == "witness" else [0] * n for t in kinds]
    return sc, [mont(s, R) for s in sc]


@pytest.mark.parametrize("group", [1, 2, 6])
def test_sort_k19_batch_group(h2b, k19_columns, group):
    k = 19
    n = 1 << k
    a0, delta = 123, 456
    sc, cols = k19_columns
    c = h2b.Context(0)
    c.set_option("msm.batch_group", group)
    try:
        params = h2b.ParamsKZG(c, k, g=bases(c, n, a0, delta))
        try:
            outs = params.commit_batch([0] * len(cols), cols)
            got = [affine(c, o) for o in outs]
        finally:
            params.close()
    finally:
        c.close()
    for j in range(len(cols)):
        assert got[j] == closed_form(sc[j], a0, delta), j
