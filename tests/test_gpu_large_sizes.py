"""Exact parity above 2^19, where several kernels take a second code path that the smaller sizes of test_gpu_parity.py
and test_gpu_prover.py never reach:
 - k_gp_scan folds more than one tile total per thread once a grand product has more than 256 tiles of 2048 (n > 2^19);
 - k_batch_invert gives every thread E > 2 elements once n exceeds one wave of 1024 slots per SM (E = 16 from 2^21);
 - the batched evaluation has more than one tile above n = 2048 and more than one tile value per thread above 2^19;
 - the product columns use the split power table (lo_bits = 10) above k = 10 and span many tiles;
 - the NTT runs its non-last pass with cw_log = 0 at 2^22 only, and three passes from 2^23 to 2^25;
 - a resident proof at k = 21 with d = 5 transforms on a 2^23 extended domain.
Every comparison is bit-exact against the oracle's C routines (oracle/bn254_oracle.c), and at k = 12 also against plain
Python integers."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *
import bench
import prover_check as pc

pytestmark = pytest.mark.gpu
R = pyref.R
ONE = mont([1], R)[0]
vp = C.c_void_p
SCAN_SIZES = [(1 << 19) + 1, (1 << 21) + 3, (1 << 23) + 5]


@pytest.fixture(scope="module")
def env():
    import torch
    import halo2_lib_b200 as h
    ctx = h.Context(0)
    yield h, ctx, torch
    ctx.close()


_residues = bench.uniform_residues  # n uniform values < 2^252 < r: valid Montgomery residues


def _to_dev(torch, a):
    """the library runs on its own non-blocking stream: torch's work on a buffer must be finished before a call reads it"""
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def _empty_dev(torch, n):
    """an output buffer: no torch kernel writes it, so nothing can land after the library's writes"""
    return torch.empty((n, 4), dtype=torch.int64, device="cuda")


def _to_host(t):
    return t.cpu().numpy().view(np.uint64)


def _tile(v, n):
    return np.tile(np.asarray(v, dtype=np.uint64).reshape(1, 4), (n, 1))


def _elements_per_thread(n, sms):
    """E of batch_invert_run: one wave of 4 CTAs of 256 threads per SM, clamped to [2, 16]"""
    slots = 256 * 4 * sms
    return min(16, max(2, -(-n // slots)))


def _powers(w, n):
    """[w^0 .. w^(n-1)] as Montgomery limbs, by doubling with the oracle's multiplier"""
    out = np.empty((n, 4), dtype=np.uint64)
    out[0] = ONE
    have = 1
    while have < n:
        m = min(have, n - have)
        out[have:have + m] = orc.f_mul(orc.FR, out[:m], _tile(mont([pow(w, have, R)], R)[0], m))
        have += m
    return out


# ------------------------------------------------------------------ scans: batch inversion and grand product
def test_scan_sizes_reach_many_elements_per_thread(env):
    """the sizes below give every batch-inversion thread more than 2 elements, and the largest reach the cap of 16"""
    h, ctx, torch = env
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    es = [_elements_per_thread(n, sms) for n in SCAN_SIZES]
    assert min(es) >= 3 and max(es) == 16, (sms, es)
    # the grand products span more than 256 tiles of 2048: every k_gp_scan thread folds several tile totals
    assert all(-(-n // 2048) > 256 for n in SCAN_SIZES)


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_batch_invert_many_elements_per_thread(env, n):
    h, ctx, torch = env
    from halo2_lib_b200._capi import lib
    E = _elements_per_thread(n, torch.cuda.get_device_properties(0).multi_processor_count)
    cta = 256 * E  # each CTA owns this many contiguous elements
    rng = np.random.default_rng(0xB2006000 + n % 1000)
    A = _residues(rng, n)
    A[::7] = 0                                   # zeros are skipped by BatchInvert::batch_invert
    c = (n // cta) // 2
    A[c * cta:(c + 1) * cta] = 0                 # one CTA with nothing to invert
    A[-1] = 0                                    # a zero last element (in the partial last CTA)
    want = orc.batch_invert(A)
    assert not want[c * cta:(c + 1) * cta].any() and want[(c - 1) * cta:c * cta].any() and want[(c + 1) * cta:].any()
    assert np.array_equal(ctx.batch_invert(A), want)
    d = _to_dev(torch, A)
    ctx.check(lib.h2b_batch_invert_fr_dev(ctx.h, vp(d.data_ptr()), n))
    ctx.synchronize()
    assert np.array_equal(_to_host(d), want)
    # an all-zero column stays zero
    d.zero_()
    torch.cuda.synchronize()
    ctx.check(lib.h2b_batch_invert_fr_dev(ctx.h, vp(d.data_ptr()), n))
    ctx.synchronize()
    assert not d.any().item()
    assert not ctx.batch_invert(np.zeros((n, 4), dtype=np.uint64)).any()


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_grand_product_many_tiles_per_thread(env, n):
    """257, 1025 and 4097 tiles: 2, 5 and 17 tile totals per k_gp_scan thread, the last thread's range partial.  With 2
    per thread the running product after the second total is never stored, so only the larger sizes check that the
    running product advances by the right tile"""
    h, ctx, torch = env
    from halo2_lib_b200._capi import lib
    rng = np.random.default_rng(0xB2006100 + n % 1000)
    F = _residues(rng, n)
    start = _residues(rng, 1)[0]
    want = orc.grand_product(F, start)
    assert np.array_equal(ctx.grand_product(F, start), want)
    d_f = _to_dev(torch, F)
    d_z = _empty_dev(torch, n)
    ctx.check(lib.h2b_grand_product_fr_dev(ctx.h, vp(d_f.data_ptr()), vp(start.ctypes.data), n, vp(d_z.data_ptr())))
    ctx.synchronize()
    assert np.array_equal(_to_host(d_z), want)


# ------------------------------------------------------------------ batched polynomial evaluation
@pytest.mark.parametrize("m,n", [(1, 1), (3, 2049), (25, (1 << 19) + 1), (40, (1 << 21) + 3)])
def test_eval_polynomial_batch_many_tiles(env, m, n):
    """(40, 2^21 + 3): 1025 tiles, 5 tile values per scan thread and a partial last thread; points 0, 1 and x * omega^r,
    and fewer polynomials than pairs, so pointers repeat inside one call"""
    h, ctx, torch = env
    from halo2_lib_b200._capi import lib
    rng = np.random.default_rng(0xB2006200 + m)
    npolys = max(1, min(m - 1, 4))
    hosts = [_residues(rng, n) for _ in range(npolys)]
    devs = [_to_dev(torch, a) for a in hosts]
    k = max(1, (n - 1).bit_length())
    w = pyref.omega_for(k)
    pts, which = [], []
    for j in range(m):
        which.append(j % npolys)
        kind = j % 3
        pts.append(0 if kind == 1 else 1 if kind == 2 else rand_ints(rng, 1, R)[0] * pow(w, int(rng.integers(0, 1 << k)), R) % R)
    xs = mont(pts, R)
    ptrs = (vp * m)(*[devs[i].data_ptr() for i in which])
    out = np.full((m, 4), 0xAB, dtype=np.uint64)
    ctx.check(lib.h2b_eval_polynomial_batch_dev(ctx.h, ptrs, vp(xs.ctypes.data), m, n, vp(out.ctypes.data)))
    for j in range(m):
        assert np.array_equal(out[j], orc.eval_polynomial(hosts[which[j]], xs[j])), j
    if n < 4096:  # plain Python integers
        for j in range(m):
            assert unmont(out[j:j + 1], R) == [pc.horner(hosts[which[j]], pts[j])], j


def test_eval_polynomial_batch_limits(env):
    h, ctx, torch = env
    from halo2_lib_b200._capi import lib
    rng = np.random.default_rng(0xB2006300)
    n = 5
    a = _residues(rng, n)
    d = _to_dev(torch, a)

    def run(m, nn, ptr_list=None):
        xs = _residues(rng, m)
        ptrs = (vp * m)(*(ptr_list if ptr_list is not None else [d.data_ptr()] * m))
        out = np.full((m, 4), 0xAB, dtype=np.uint64)
        ctx.check(lib.h2b_eval_polynomial_batch_dev(ctx.h, ptrs, vp(xs.ctypes.data), m, nn, vp(out.ctypes.data)))
        return xs, out
    xs, out = run(4096, n)  # the largest batch accepted
    for j in range(4096):
        assert np.array_equal(out[j], orc.eval_polynomial(a, xs[j])), j
    with pytest.raises(h.H2BError):
        run(4097, n)
    xs, out = run(3, 0)  # empty polynomials evaluate to zero
    assert not out.any()
    with pytest.raises(h.H2BError):
        run(3, n, [d.data_ptr(), None, d.data_ptr()])


# ------------------------------------------------------------------ product columns
PERM_SETS = [(0, 3), (3, 8), (11, 1)]  # (first column, columns): halo2 chains the sets through z[u]


def _perm_factors(cols, sig, beta, gamma, k, sets):
    """per set, the row factors prod_j (v_j + beta delta^j omega^i + gamma) / prod_j (v_j + beta sigma_j(i) + gamma) on
    every row (a zero denominator gives 0, as BatchInvert leaves zeros alone), oracle field ops"""
    n = 1 << k
    W = _powers(pyref.omega_for(k), n)
    G, B = _tile(mont([gamma], R)[0], n), _tile(mont([beta], R)[0], n)
    out = []
    for first, cnt in sets:
        num = den = None
        for j in range(first, first + cnt):
            bd = _tile(mont([beta * pow(pyref.DELTA, j, R) % R], R)[0], n)
            t_num = orc.f_add(orc.FR, orc.f_add(orc.FR, cols[j], orc.f_mul(orc.FR, W, bd)), G)
            t_den = orc.f_add(orc.FR, orc.f_add(orc.FR, cols[j], orc.f_mul(orc.FR, sig[j], B)), G)
            num = t_num if num is None else orc.f_mul(orc.FR, num, t_num)
            den = t_den if den is None else orc.f_mul(orc.FR, den, t_den)
        out.append(orc.f_mul(orc.FR, num, orc.batch_invert(den)))
    return out


def _chain(factors, u, starts_first=ONE):
    """z of every set: rows >= u have factor 1, each set starts from the previous set's z[u]"""
    zs, start = [], starts_first
    for f in factors:
        f = f.copy()
        f[u:] = ONE
        z = orc.grand_product(f, start)
        zs.append(z)
        start = z[u]
    return zs


def _perm_z_ints(cols, sig, beta, gamma, k, u, sets):
    """the same recurrence on plain Python integers"""
    n = 1 << k
    w = pyref.omega_for(k)
    wi = [pow(w, i, R) for i in range(n)]
    dj = [pow(pyref.DELTA, j, R) for j in range(len(cols))]
    zs, carry = [], 1
    for first, cnt in sets:
        z = [carry]
        for i in range(n - 1):
            f = 1
            if i < u:
                num = den = 1
                for j in range(first, first + cnt):
                    num = num * (cols[j][i] + beta * dj[j] * wi[i] + gamma) % R
                    den = den * (cols[j][i] + beta * sig[j][i] + gamma) % R
                f = num * pow(den, -1, R) % R if den else 0
            z.append(z[-1] * f % R)
        carry = z[u]
        zs.append(z)
    return zs


@pytest.mark.parametrize("k", [12, 21])
def test_permutation_product_chained_sets(env, k):
    """3 + 8 + 1 columns in three chained sets; u on a 2048-row tile boundary and one row either side; one row of the last
    set has a zero denominator (sigma = -(v + gamma) / beta), so its factor is 0 and the rest of that set is 0"""
    h, ctx, torch = env
    from halo2_lib_b200._capi import lib
    n = 1 << k
    ncols = 12
    rng = np.random.default_rng(0xB2006400 + k)
    beta, gamma = rand_ints(rng, 2, R)
    bl, gl = mont([beta], R)[0], mont([gamma], R)[0]
    cols = [_residues(rng, n) for _ in range(ncols)]
    sig = [_residues(rng, n) for _ in range(ncols)]
    r0 = n - 2049 - 7  # below every u tried
    v = unmont(cols[11][r0:r0 + 1], R)[0]
    sig[11][r0] = mont([-(v + gamma) * pow(beta, -1, R) % R], R)[0]
    d_cols = [_to_dev(torch, c) for c in cols]
    d_sig = [_to_dev(torch, s) for s in sig]
    d_z = [_empty_dev(torch, n) for _ in PERM_SETS]
    factors = _perm_factors(cols, sig, beta, gamma, k, PERM_SETS)
    assert not factors[2][r0].any()

    def run(bf, sets=PERM_SETS, z=d_z):
        for s, (first, cnt) in enumerate(sets):
            tc = (vp * max(cnt, 1))(*[d_cols[j].data_ptr() for j in range(first, first + cnt)])
            ts = (vp * max(cnt, 1))(*[d_sig[j].data_ptr() for j in range(first, first + cnt)])
            start = vp(z[s - 1].data_ptr() + 32 * (n - (bf + 1))) if s else None
            ctx.check(lib.h2b_permutation_product_dev(ctx.h, tc, ts, cnt, first, vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf, start,
                                                      vp(z[s].data_ptr())))
        ctx.synchronize()
        return [_to_host(t) for t in z]

    for bf in (2047, 2046, 2048):  # u = n - 2048 is a multiple of the 2048-row tile
        u = n - (bf + 1)
        got = run(bf)
        want = _chain(factors, u)
        for s in range(len(PERM_SETS)):
            assert np.array_equal(got[s], want[s]), (bf, s)
            assert (got[s][u + 1:] == got[s][u]).all(), (bf, s)
        assert got[0][u].any() and got[1][u].any() and not got[2][r0 + 1:].any() and got[2][r0].any()
        if k == 12 and bf == 2047:
            ints = _perm_z_ints([unmont(c, R) for c in cols], [unmont(s, R) for s in sig], beta, gamma, k, u, PERM_SETS)
            for s in range(len(PERM_SETS)):
                assert unmont(got[s], R) == ints[s], s
    for cnt in (0, 9):  # 1..8 columns per set
        with pytest.raises(h.H2BError):
            run(2047, [(0, cnt)])
    with pytest.raises(h.H2BError):  # no usable rows
        run(n - 1, [(0, 3)])


@pytest.mark.parametrize("k", [12, 21])
def test_lookup_product_and_elementwise_mul(env, k):
    h, ctx, torch = env
    from halo2_lib_b200._capi import lib
    n = 1 << k
    rng = np.random.default_rng(0xB2006500 + k)
    beta, gamma = rand_ints(rng, 2, R)
    bl, gl = mont([beta], R)[0], mont([gamma], R)[0]
    inp, tab, pin, ptab = (_residues(rng, n) for _ in range(4))
    r0 = n - 2049 - 3
    pin[r0] = mont([R - beta], R)[0]  # (permuted input + beta) = 0 on one row: factor 0
    dev = [_to_dev(torch, a) for a in (inp, tab, pin, ptab)]
    d_z = _empty_dev(torch, n)
    G, B = _tile(gl, n), _tile(bl, n)
    num = orc.f_mul(orc.FR, orc.f_add(orc.FR, inp, B), orc.f_add(orc.FR, tab, G))
    den = orc.f_mul(orc.FR, orc.f_add(orc.FR, pin, B), orc.f_add(orc.FR, ptab, G))
    f_all = orc.f_mul(orc.FR, num, orc.batch_invert(den))
    assert not f_all[r0].any()
    for bf in (2047, 2046, 2048):
        u = n - (bf + 1)
        ctx.check(lib.h2b_lookup_product_dev(ctx.h, *[vp(t.data_ptr()) for t in dev], vp(bl.ctypes.data), vp(gl.ctypes.data), k, bf,
                                             vp(d_z.data_ptr())))
        ctx.synchronize()
        got = _to_host(d_z)
        assert np.array_equal(got, _chain([f_all], u)[0]), bf
        assert got[r0].any() and not got[r0 + 1:].any()
        if k == 12 and bf == 2047:
            a, t, pa, pt = (unmont(x, R) for x in (inp, tab, pin, ptab))
            z = [1]
            for i in range(n - 1):
                f = 1
                if i < u:
                    d = (pa[i] + beta) * (pt[i] + gamma) % R
                    f = (a[i] + beta) * (t[i] + gamma) % R * (pow(d, -1, R) if d else 0) % R
                z.append(z[-1] * f % R)
            assert unmont(got, R) == z
    with pytest.raises(h.H2BError):
        ctx.check(lib.h2b_lookup_product_dev(ctx.h, *[vp(t.data_ptr()) for t in dev], vp(bl.ctypes.data), vp(gl.ctypes.data), k, n - 1,
                                             vp(d_z.data_ptr())))
    # h2b_fr_mul_elementwise_dev: separate output and output aliased to a
    for m in (1, 257) + (((1 << 21) + 1,) if k == 21 else ()):
        a, b = _residues(rng, m), _residues(rng, m)
        want = orc.f_mul(orc.FR, a, b)
        da, db, do = _to_dev(torch, a), _to_dev(torch, b), _empty_dev(torch, m)
        ctx.check(lib.h2b_fr_mul_elementwise_dev(ctx.h, vp(da.data_ptr()), vp(db.data_ptr()), m, vp(do.data_ptr())))
        ctx.check(lib.h2b_fr_mul_elementwise_dev(ctx.h, vp(da.data_ptr()), vp(db.data_ptr()), m, vp(da.data_ptr())))
        ctx.synchronize()
        assert np.array_equal(_to_host(do), want) and np.array_equal(_to_host(da), want), m
        if m == 257:
            assert unmont(want, R) == [x * y % R for x, y in zip(unmont(a, R), unmont(b, R))]


# ------------------------------------------------------------------ NTT at 2^22 .. 2^25
@pytest.mark.parametrize("log_n", [22, 23, 24, 25])
def test_ntt_forward_exact(env, log_n):
    """2^22: both radix digits are 11, the non-last pass runs with cw_log = 0; 2^23 .. 2^25: three passes"""
    h, ctx, torch = env
    n = 1 << log_n
    A = _residues(np.random.default_rng(0xB2006600 + log_n), n)
    w = orc.omega(log_n)
    assert np.array_equal(h.best_fft(ctx, A, w, log_n), orc.ntt_fast(A, log_n, w))


@pytest.mark.parametrize("k", [22, 23])
def test_lagrange_to_coeff_exact(env, k):
    h, ctx, torch = env
    A = _residues(np.random.default_rng(0xB2006700 + k), 1 << k)
    orc.use_fast_ntt(True)
    try:
        want = orc.lagrange_to_coeff(A, k)
    finally:
        orc.use_fast_ntt(False)
    assert np.array_equal(h.EvaluationDomain(ctx, 3, k).lagrange_to_coeff(A), want)


@pytest.mark.parametrize("k,j", [(21, 5), (23, 4)])
def test_coset_transforms_exact(env, k, j):
    h, ctx, torch = env
    n = 1 << k
    A = _residues(np.random.default_rng(0xB2006800 + k), n)
    dom = h.EvaluationDomain(ctx, j, k)
    assert dom.extended_k == k + 2
    ext = dom.coeff_to_extended(A)
    orc.use_fast_ntt(True)
    try:
        assert np.array_equal(ext, orc.coeff_to_extended(A, dom.extended_k))
        back = dom.extended_to_coeff(ext)
        assert np.array_equal(back, orc.extended_to_coeff(ext, dom.extended_k)[: n * (j - 1)])
    finally:
        orc.use_fast_ntt(False)
    assert np.array_equal(back[:n], A) and not back[n:].any()


def test_ntt_max_ctas_per_sm_does_not_change_results(env):
    """the option ntt.max_ctas_per_sm only limits how many CTAs of a transform share an SM: outputs are byte-identical
    to a context without it, forward, inverse and coset forms, one to three passes"""
    h, ctx, torch = env
    rng = np.random.default_rng(0xB2006900)
    fwd = {}
    for log_n in (12, 22, 23):
        A = _residues(rng, 1 << log_n)
        fwd[log_n] = (A, h.best_fft(ctx, A, h.omega(log_n), log_n))
    inv22 = h.EvaluationDomain(ctx, 3, 22).lagrange_to_coeff(fwd[22][0])
    coset = {}
    for k in (12, 21):
        A = _residues(rng, 1 << k)
        ext = h.EvaluationDomain(ctx, 5, k).coeff_to_extended(A)
        coset[k] = (A, ext, h.EvaluationDomain(ctx, 5, k).extended_to_coeff(ext))
    c2 = h.Context(0)
    try:
        with pytest.raises(h.H2BError):
            c2.set_option("ntt.max_ctas_per_sm", 3)
        for v in (1, 2):
            c2.set_option("ntt.max_ctas_per_sm", v)
            for log_n, (A, F) in fwd.items():
                assert np.array_equal(h.best_fft(c2, A, h.omega(log_n), log_n), F), (v, log_n)
            assert np.array_equal(h.EvaluationDomain(c2, 3, 22).lagrange_to_coeff(fwd[22][0]), inv22), v
            for k, (A, ext, back) in coset.items():
                dom = h.EvaluationDomain(c2, 5, k)
                assert np.array_equal(dom.coeff_to_extended(A), ext), (v, k)
                assert np.array_equal(dom.extended_to_coeff(ext), back), (v, k)
    finally:
        c2.close()


# ------------------------------------------------------------------ a resident proof at k = 21
def _progression_bases_dev(ctx, torch, n, a0, delta):
    """b_i = (a0 + i * delta) * G on the device"""
    from halo2_lib_b200._capi import lib
    g = affine_to_limbs([pyref.G1])[0]
    sc = np.zeros((n, 4), dtype=np.uint64)
    sc[:, 0] = a0 + delta * np.arange(n, dtype=np.uint64)
    d_sc = _to_dev(torch, ctx.field_op(1, 5, sc))
    d_pts = torch.empty((n, 8), dtype=torch.int64, device="cuda")
    ctx.check(lib.h2b_g1_fixed_base_mul_dev(ctx.h, vp(g.ctypes.data), vp(d_sc.data_ptr()), n, vp(d_pts.data_ptr())))
    ctx.synchronize()
    return d_pts


def _prove(sess, inst, rnd, virtual=None):
    v = np.ascontiguousarray(inst["virtual"] if virtual is None else virtual)
    lk = np.ascontiguousarray(inst["lookup"])
    return sess.prove(v.ctypes.data, len(v), rnd.ctypes.data, seed=5, break_points=inst["break_points"],
                      lookup_ptr=lk.ctypes.data if len(lk) else 0, n_lookup=len(lk))


@pytest.mark.parametrize("A,L", [(1, 0), (3, 2)], ids=["selector_lookup_d5", "chained_sets_two_lookups"])
def test_resident_proof_k21(env, A, L):
    """A = 1, L = 0 with the selector lookup is the ECDSA / pairing shape (degree 5, extended domain 2^23); A = 3, L = 2
    has three chained permutation sets and two lookups"""
    h, ctx, torch = env
    k = 21
    n = 1 << k
    prog = {0: (3, 5), 1: (7, 11)}  # basis -> (a0, delta) of its progression a_i * G
    d_m = _progression_bases_dev(ctx, torch, n, *prog[0])
    d_l = _progression_bases_dev(ctx, torch, n, *prog[1])
    params = h.ParamsKZG(ctx, k, g=d_m.data_ptr(), g_lagrange=d_l.data_ptr(), device_ptrs=True)
    rng = np.random.default_rng(0xB2006A00 + A)
    inst = h.synthetic_circuit(ctx, k, rng, A=A, L=L, selector_lookup=True)
    cs = h.Circuit(ctx, k, inst["fixed"], inst["sigma"], A=A, L=L, selector_lookup=True)
    assert cs.ext_k == 23 and cs.degree == (5 if L == 0 else 4) and cs.n_sets == (1 if L == 0 else 3)
    sess = h.ProverSession(ctx, params, cs)
    rnd = _residues(rng, n)
    sess.keep = {}
    res = _prove(sess, inst, rnd)
    kept, sess.keep = sess.keep["committed"], None
    nlk = cs.n_lookups
    assert len(res["commitments"]) == len(kept) == (A + L) + 2 * nlk + (cs.n_sets + nlk + 1) + (cs.degree - 1) + 2
    for j, (cm, (basis, poly)) in enumerate(zip(res["commitments"], kept)):
        a0, d = prog[basis]
        s = bench.progression_dot(poly, a0, d, 0) * bench.MONT_RINV_R % R
        assert jac_limbs_to_affine(cm) == (pyref.g1_mul(s, pyref.G1) if s else None), j
    left, right = pc.quotient_identity(res, k, cs.bf, A, L, True)
    assert left == right
    x = res["challenges"]["x"]
    w = pyref.omega_for(k)

    def check_eval(name, rot, coeffs):
        want = orc.eval_polynomial(coeffs, mont([x * pow(w, rot % n, R) % R], R)[0])
        assert np.array_equal(np.asarray(res["evals"][(name, rot)], dtype=np.uint64).reshape(4), want), (name, rot)
    check_eval("a0", 2, sess.coef["a0"].download())
    check_eval("zp0", 1, sess.coef["zp0"].download())
    check_eval("zl0", 1, sess.coef["zl0"].download())
    if cs.n_sets > 1:
        check_eval("zp0", -(cs.bf + 1), sess.coef["zp0"].download())
    for j in range(cs.degree - 1):
        check_eval("h%d" % j, 0, sess.h.download(j * n, n))
    # a broken gate on the same session: the identity must fail
    bad = np.ascontiguousarray(inst["virtual"]).copy()
    bad[3] = mont([12345], R)[0]
    res2 = _prove(sess, inst, rnd, virtual=bad)
    l2, r2 = pc.quotient_identity(res2, k, cs.bf, A, L, True)
    assert l2 != r2
    sess.free(); cs.free(); params.close()
    del d_m, d_l
