"""GPU parity at BASELINE.json's full sizes (k = 19, 20, 23; extended domains up to 2^25) through size-independent
properties: closed forms, linearity, round trips and agreement between independent device paths (fixed-base table vs
ad-hoc windows).  All comparisons are exact.  Element-by-element parity with the oracle at these sizes is in
test_gpu_large_sizes.py."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *

pytestmark = pytest.mark.gpu
R = pyref.R


@pytest.fixture(scope="module")
def env():
    import torch
    import halo2_lib_b200 as h
    ctx = h.Context(0)
    yield h, ctx, torch
    ctx.close()


def _uniform(rng, n):
    a = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.int64).astype(np.uint64)
    a[:, 3] &= np.uint64((1 << 60) - 1)
    return a


def _ints_from_limbs(a):
    """vectorised limbs -> python ints (object array)"""
    a = a.astype(object)
    return a[:, 0] + (a[:, 1] << 64) + (a[:, 2] << 128) + (a[:, 3] << 192)


def _progression_bases_dev(h, ctx, torch, n, a0, delta):
    from halo2_lib_b200._capi import lib
    g = affine_to_limbs([pyref.G1])[0]
    sc = np.zeros((n, 4), dtype=np.uint64)
    sc[:, 0] = a0 + delta * np.arange(n, dtype=np.uint64)
    d_sc = torch.from_numpy(ctx.field_op(1, 5, sc).view(np.int64)).cuda()
    d_pts = torch.empty((n, 8), dtype=torch.int64, device="cuda")
    ctx.check(lib.h2b_g1_fixed_base_mul_dev(ctx.h, C.c_void_p(g.ctypes.data), C.c_void_p(d_sc.data_ptr()), n, C.c_void_p(d_pts.data_ptr())))
    ctx.synchronize()
    return d_pts


@pytest.mark.parametrize("k", [19, 20, 23])
def test_msm_closed_form_full_size(env, k):
    """bases a_i*G with a_i = a0 + i*delta (canonical < 2^64)  =>  commit(s) == (sum s_i a_i mod r) * G"""
    h, ctx, torch = env
    n = 1 << k
    a0, delta = 1234567, 89
    d_pts = _progression_bases_dev(h, ctx, torch, n, a0, delta)
    params = h.ParamsKZG(ctx, k, g=d_pts.data_ptr(), device_ptrs=True)
    rng = np.random.default_rng(0xB2000000 + k)
    half = n // 2
    import bench
    S_canon = np.concatenate([_uniform(rng, half), bench.witness_like(rng, n - half)])  # canonical values
    S = ctx.field_op(1, 5, S_canon)  # to Montgomery on the GPU (checked against the oracle in test_gpu_parity)
    got = jac_limbs_to_affine(ctx.g1_normalize(params.commit(S).reshape(1, 12))[0])
    a = a0 + delta * np.arange(n, dtype=object)
    kk = int((_ints_from_limbs(S_canon) * a).sum() % R)
    assert got == pyref.g1_mul(kk, pyref.G1)
    # independent device path on a slice: ad-hoc windows (no table) on the first 2^16 points
    m = 1 << 16
    bases_host = d_pts[:m].cpu().numpy().view(np.uint64)
    adhoc = jac_limbs_to_affine(ctx.g1_normalize(h.best_multiexp(ctx, S[:m], bases_host).reshape(1, 12))[0])
    kk2 = int((_ints_from_limbs(S_canon[:m]) * a[:m]).sum() % R)
    assert adhoc == pyref.g1_mul(kk2, pyref.G1)
    params.close()
    del d_pts


def test_grouped_commitment_phase_full_size(env):
    """the advice phase of the k = 20 MSM-circuit config (halo2-ecc/configs/bn254/bench_msm.config:5: 11 + 2 advice
    columns => 13 commitments in one batch call) plus monomial-basis columns in the same call: the grouped pipelines
    (bucket sets side by side, table bit in the sorted entries) at full size, every commitment against its closed form"""
    h, ctx, torch = env
    import bench
    k = 20
    n = 1 << k
    prog = {0: (1234567, 89), 1: (7654321, 97)}  # basis -> (a0, delta) of its progression a_i * G
    d_m = _progression_bases_dev(h, ctx, torch, n, *prog[0])
    d_l = _progression_bases_dev(h, ctx, torch, n, *prog[1])
    params = h.ParamsKZG(ctx, k, g=d_m.data_ptr(), g_lagrange=d_l.data_ptr(), device_ptrs=True)
    rng = np.random.default_rng(0xB2004000)
    basis = [1] * 13 + [0, 1, 0]
    cols, d_cols = [], []
    for j in range(len(basis)):
        canon = bench.witness_like(rng, n) if j % 3 else _uniform(rng, n)
        if j == 5:
            canon[:] = 0  # an all-zero column inside the group
        S = ctx.field_op(1, 5, canon)
        cols.append(S)
        d_cols.append(torch.from_numpy(S.view(np.int64)).cuda())
    d_out = torch.zeros((len(basis), 12), dtype=torch.int64, device="cuda")
    params.commit_batch_dev(basis, [t.data_ptr() for t in d_cols], n, d_out.data_ptr())
    torch.cuda.synchronize()
    outs = ctx.g1_normalize(d_out.cpu().numpy().view(np.uint64))
    for j, b in enumerate(basis):
        a0, d = prog[b]
        kk = bench.progression_dot(cols[j], a0, d, 0) * bench.MONT_RINV_R % R
        want = pyref.g1_mul(kk, pyref.G1) if kk else None
        assert jac_limbs_to_affine(outs[j]) == want, j
    params.close()
    del d_m, d_l, d_cols


@pytest.mark.parametrize("k", [19, 23, 25])
def test_ntt_properties_full_size(env, k):
    h, ctx, torch = env
    n = 1 << k
    rng = np.random.default_rng(0xB2001000 + k)
    A = _uniform(rng, n)
    w = h.omega(k)
    F = h.best_fft(ctx, A, w, k)
    dom = h.EvaluationDomain(ctx, 3, k)
    # round trip: lagrange_to_coeff(best_fft(A)) == A
    assert np.array_equal(dom.lagrange_to_coeff(F), A)
    # definition at a few output indices: F[i] = sum_j A[j] w^(ij)  (Horner over python ints on 2^12-strided subsample
    # is not the definition, so use linearity + a delta instead): NTT(e_j)[i] = w^(ij)
    j = int(rng.integers(1, n))
    E = np.zeros((n, 4), dtype=np.uint64)
    E[j] = mont([1], R)[0]
    Fe = h.best_fft(ctx, E, w, k)
    wk = pyref.omega_for(k)
    for i in (0, 1, 2, n // 2 + 1, n - 1, int(rng.integers(0, n))):
        assert unmont(Fe[i:i + 1], R) == [pow(wk, i * j, R)]
    # linearity: NTT(A + E) == NTT(A) + NTT(E) checked on the whole array with the oracle's field adds
    AE = orc.f_add(orc.FR, A, E)
    assert np.array_equal(h.best_fft(ctx, AE, w, k), orc.f_add(orc.FR, F, Fe))


@pytest.mark.parametrize("k,j", [(19, 5), (23, 4)])
def test_coset_round_trip_full_size(env, k, j):
    h, ctx, torch = env
    n = 1 << k
    rng = np.random.default_rng(0xB2001000 + 500 + k)
    A = _uniform(rng, n)
    dom = h.EvaluationDomain(ctx, j, k)
    ext = dom.coeff_to_extended(A)
    assert len(ext) == 1 << dom.extended_k and dom.extended_k == k + 2
    # ext[0] = a(zeta) : Horner on the host over python ints is O(n) big-int work; use the oracle's field ops on a
    # 2^14-coefficient polynomial embedded in the same domain instead (zero-padded), exact definition check
    small = 1 << 14
    B = A[:small]
    ext_b = h.EvaluationDomain(ctx, j, k).coeff_to_extended(np.concatenate([B, np.zeros((n - small, 4), dtype=np.uint64)]))
    b = unmont(B, R)
    we = pyref.omega_for(dom.extended_k)
    for i in (0, 5, (1 << dom.extended_k) - 1):
        x = pyref.ZETA * pow(we, i, R) % R
        acc = 0
        for c in reversed(b):
            acc = (acc * x + c) % R
        assert unmont(ext_b[i:i + 1], R) == [acc]
    back = dom.extended_to_coeff(ext)
    assert np.array_equal(back[:n], A) and not back[n:].any()


def test_assignment_full_size(env):
    """k = 20, 11 columns (halo2-ecc/configs/bn254/bench_msm.config:5 shape): closed form of the walk on 1.1e7 cells"""
    h, ctx, torch = env
    k, ncols = 20, 11
    rows = 1 << k
    max_rows = rows - 20
    rng = np.random.default_rng(77)
    N = 10 * (max_rows - 1) + 12345
    V = _uniform(rng, N)
    bps = [max_rows - 1 - int(x) for x in rng.integers(0, 3, size=10)]  # break rows as assign_with_constraints would pin them
    cols = h.assign_witnesses(ctx, [V[:1000], V[1000:N // 2], V[N // 2:]], bps, k, ncols)
    s = 0
    for c, b in enumerate(bps):
        assert np.array_equal(cols[c, : b + 1], V[s : s + b + 1])
        assert not cols[c, b + 1 :].any()
        s += b
    last = N - s
    assert np.array_equal(cols[10, :last], V[s:]) and not cols[10, last:].any()
