"""GPU tests of the C ABI's twins (-m gpu): every entry point of include/h2b200.h that has a host-pointer form and a `_dev`
form is run both ways on the same seeded inputs and must give byte-identical outputs, empty inputs included wherever the
ABI allows them.  The batch transforms are held against the single `_dev` transforms, and SRS handles from host and
device bases against each other through their commitments.  Bad arguments (null pointers, k / ext_k out of range) must
return the same status code in both forms and leave the context usable."""
import ctypes as C
import numpy as np
import pytest
from oracle import pyref
from util import mont, rand_ints, affine_to_limbs

pytestmark = pytest.mark.gpu
R = pyref.R
OK, ARG, UNSATISFIED = 0, -1, -5
vp = C.c_void_p


@pytest.fixture(scope="module")
def env():
    import torch
    import halo2_lib_b200 as h
    from halo2_lib_b200._capi import lib
    ctx = h.Context(0)
    yield ctx, lib, torch
    ctx.close()


def fr(seed, n):
    return mont(rand_ints(np.random.default_rng(seed), n, R), R)


def hp(a):
    """host pointer of a numpy array (null for None)"""
    return None if a is None else vp(a.ctypes.data)


class Dev:
    """device copies of host arrays for the `_dev` forms; the context's stream is joined before anything is read back"""

    def __init__(self, env):
        self.ctx, self.lib, self.torch = env
        self.keep = []

    def put(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a).view(np.int64).reshape(-1).copy()).cuda()
        self.keep.append(t)
        self.torch.cuda.synchronize()
        return vp(t.data_ptr()) if t.numel() else None, t

    def zeros(self, words):
        t = self.torch.zeros(max(words, 1), dtype=self.torch.int64, device="cuda")
        self.keep.append(t)
        self.torch.cuda.synchronize()
        return vp(t.data_ptr()), t

    def get(self, t, words=None):
        self.ctx.synchronize()
        return t.cpu().numpy().view(np.uint64)[:words]


def points(env, seed, n):
    """n affine points (n x 8 Montgomery limbs), none of them the identity"""
    ctx = env[0]
    return ctx.g1_fixed_base_mul(affine_to_limbs([pyref.G1])[0], fr(seed, n) | np.uint64(1))


def xyz(pts):
    one = mont([1], pyref.P)[0]
    return np.concatenate([pts, np.tile(one, (len(pts), 1))], axis=1)


# ------------------------------------------------------------------------------------------------ transforms
@pytest.mark.parametrize("log_n,scale", [(0, 0), (5, 1), (10, 0)])
def test_ntt_fr(env, log_n, scale):
    ctx, lib, _ = env
    d = Dev(env)
    a = fr(10 + log_n, 1 << log_n)
    w = np.zeros(4, dtype=np.uint64)
    assert lib.h2b_domain_omega(log_n, hp(w)) == OK
    host = a.copy()
    ctx.check(lib.h2b_ntt_fr(ctx.h, hp(host), log_n, hp(w), scale))
    p, t = d.put(a)
    ctx.check(lib.h2b_ntt_fr_dev(ctx.h, p, log_n, hp(w), scale))
    assert np.array_equal(d.get(t), host.reshape(-1))


@pytest.mark.parametrize("name", ["lagrange_to_coeff", "coeff_to_lagrange", "extended_to_coeff"])
@pytest.mark.parametrize("k", [0, 7])
def test_domain_transforms(env, name, k):
    ctx, lib, _ = env
    d = Dev(env)
    a = fr(20 + k, 1 << k)
    host = a.copy()
    ctx.check(getattr(lib, "h2b_" + name)(ctx.h, hp(host), k))
    p, t = d.put(a)
    ctx.check(getattr(lib, "h2b_" + name + "_dev")(ctx.h, p, k))
    assert np.array_equal(d.get(t), host.reshape(-1))


@pytest.mark.parametrize("n_coeffs,ext_k", [(0, 3), (50, 7), (128, 7)])
def test_coeff_to_extended(env, n_coeffs, ext_k):
    ctx, lib, _ = env
    d = Dev(env)
    a = fr(30 + n_coeffs, n_coeffs).reshape(-1, 4)
    host = np.empty((1 << ext_k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_coeff_to_extended(ctx.h, hp(a), n_coeffs, ext_k, hp(host)))
    p, _ = d.put(a)
    po, to = d.zeros(4 << ext_k)
    ctx.check(lib.h2b_coeff_to_extended_dev(ctx.h, p if n_coeffs else po, n_coeffs, ext_k, po))
    assert np.array_equal(d.get(to), host.reshape(-1))


def _ptrs(arrs):
    return (C.c_void_p * max(len(arrs), 1))(*[a.ctypes.data for a in arrs])


@pytest.mark.parametrize("m", [0, 1, 4])
def test_batch_transforms_match_the_dev_transforms(env, m):
    ctx, lib, _ = env
    d = Dev(env)
    k, ext_k, n_coeffs = 5, 7, 40
    cols = [fr(40 + j, 1 << k) for j in range(m)]

    def single(name, a, *args):
        p, t = d.put(a)
        ctx.check(getattr(lib, name)(ctx.h, p, *args))
        return d.get(t)

    for name in ("lagrange_to_coeff", "coeff_to_lagrange"):
        host = [c.copy() for c in cols]
        ctx.check(getattr(lib, f"h2b_{name}_batch")(ctx.h, _ptrs(host), m, k))
        for c, h in zip(cols, host):
            assert np.array_equal(h.reshape(-1), single(f"h2b_{name}_dev", c, k))
    coeffs = [fr(45 + j, n_coeffs) for j in range(m)]
    out = [np.empty((1 << ext_k, 4), dtype=np.uint64) for _ in range(m)]
    ctx.check(lib.h2b_coeff_to_extended_batch(ctx.h, _ptrs(coeffs), m, n_coeffs, ext_k, _ptrs(out)))
    for c, o in zip(coeffs, out):
        p, _ = d.put(c)
        po, to = d.zeros(4 << ext_k)
        ctx.check(lib.h2b_coeff_to_extended_dev(ctx.h, p, n_coeffs, ext_k, po))
        assert np.array_equal(o.reshape(-1), d.get(to))
    a = [c.copy() for c in cols]
    ext = [np.empty((1 << ext_k, 4), dtype=np.uint64) for _ in range(m)]
    ctx.check(lib.h2b_lagrange_to_coeff_and_extended_batch(ctx.h, _ptrs(a), m, k, ext_k, _ptrs(ext)))
    for c, h, e in zip(cols, a, ext):
        coeff = single("h2b_lagrange_to_coeff_dev", c, k)
        assert np.array_equal(h.reshape(-1), coeff)
        p, _ = d.put(coeff)
        po, to = d.zeros(4 << ext_k)
        ctx.check(lib.h2b_coeff_to_extended_dev(ctx.h, p, 1 << k, ext_k, po))
        assert np.array_equal(e.reshape(-1), d.get(to))


# ------------------------------------------------------------------------------------------------ assignment and scans
@pytest.mark.parametrize("N,k,ncols,bps", [(0, 4, 2, []), (250, 6, 6, [50] * 5)])
def test_assign_columns(env, N, k, ncols, bps):
    ctx, lib, _ = env
    d = Dev(env)
    v, bp = fr(50 + N, N).reshape(-1, 4), np.array(bps, dtype=np.uint64)
    host = np.empty((ncols << k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_assign_columns(ctx.h, hp(v), N, hp(bp), len(bps), k, ncols, hp(host)))
    p, _ = d.put(v)
    po, to = d.zeros(4 * (ncols << k))
    ctx.check(lib.h2b_assign_columns_dev(ctx.h, p, N, hp(bp), len(bps), k, ncols, po))
    assert np.array_equal(d.get(to), host.reshape(-1))


@pytest.mark.parametrize("N,tags", [(0, 3), (200, 2), (200, 3)])
def test_assign_columns_assigned(env, N, tags):
    """Assigned<Fr> records (tag, numerator, denominator): Zero / Trivial only, and with Rational cells (some den = 0)"""
    ctx, lib, _ = env
    d = Dev(env)
    k, ncols, bp = 6, 6, np.array([50] * 3, dtype=np.uint64)
    rng = np.random.default_rng(60 + N + tags)
    cells = np.zeros((N, 9), dtype=np.uint64)
    cells[:, 0] = rng.integers(0, tags, size=N)
    cells[:, 1:5] = fr(61, N).reshape(-1, 4)
    cells[:, 5:9] = fr(62, N).reshape(-1, 4)
    cells[::7, 5:9] = 0
    host = np.empty((ncols << k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_assign_columns_assigned(ctx.h, hp(cells), N, hp(bp), len(bp), k, ncols, hp(host)))
    p, _ = d.put(cells)
    po, to = d.zeros(4 * (ncols << k))
    ctx.check(lib.h2b_assign_columns_assigned_dev(ctx.h, p, N, hp(bp), len(bp), k, ncols, po))
    assert np.array_equal(d.get(to), host.reshape(-1))


@pytest.mark.parametrize("N,k,L", [(0, 4, 1), (100, 6, 2)])
def test_assign_lookups(env, N, k, L):
    ctx, lib, _ = env
    d = Dev(env)
    v = fr(70 + N, N).reshape(-1, 4)
    host = np.empty((L << k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_assign_lookups(ctx.h, hp(v), N, k, L, hp(host)))
    p, _ = d.put(v)
    po, to = d.zeros(4 * (L << k))
    ctx.check(lib.h2b_assign_lookups_dev(ctx.h, p, N, k, L, po))
    assert np.array_equal(d.get(to), host.reshape(-1))


@pytest.mark.parametrize("n", [0, 1, 300])
def test_scans(env, n):
    """eval_rational, batch_invert and grand_product; zeros among the denominators / inputs"""
    ctx, lib, _ = env
    d = Dev(env)
    num, den, start = fr(80 + n, n).reshape(-1, 4), fr(81 + n, n).reshape(-1, 4), fr(82, 1)[0]
    den[::5] = 0
    outs = {}
    host = np.empty((n, 4), dtype=np.uint64)
    ctx.check(lib.h2b_eval_rational(ctx.h, hp(num), hp(den), n, hp(host)))
    (pn, _), (pd, _), (po, to) = d.put(num), d.put(den), d.zeros(4 * n)
    ctx.check(lib.h2b_eval_rational_dev(ctx.h, pn, pd, n, po if n else None))
    outs["eval_rational"] = (host, d.get(to, 4 * n))
    host = den.copy()
    ctx.check(lib.h2b_batch_invert_fr(ctx.h, hp(host), n))
    pd, td = d.put(den)
    ctx.check(lib.h2b_batch_invert_fr_dev(ctx.h, pd, n))
    outs["batch_invert"] = (host, d.get(td, 4 * n))
    host = np.empty((n, 4), dtype=np.uint64)
    ctx.check(lib.h2b_grand_product_fr(ctx.h, hp(num), hp(start), n, hp(host)))
    (pn, _), (po, to) = d.put(num), d.zeros(4 * n)
    ctx.check(lib.h2b_grand_product_fr_dev(ctx.h, pn, hp(start), n, po if n else None))
    outs["grand_product"] = (host, d.get(to, 4 * n))
    for name, (h, g) in outs.items():
        assert np.array_equal(h.reshape(-1), g), name


# ------------------------------------------------------------------------------------------------ quotient
@pytest.mark.parametrize("k,ext_k", [(4, 4), (4, 6)])
def test_flex_gate_fold(env, k, ext_k):
    ctx, lib, _ = env
    d = Dev(env)
    n = 1 << ext_k
    q, a, acc, y = fr(90, n), fr(91, n), fr(92, n), fr(93, 1)[0]
    host = acc.copy()
    ctx.check(lib.h2b_flex_gate_fold(ctx.h, hp(q), hp(a), hp(y), k, ext_k, hp(host)))
    (pq, _), (pa, _), (pacc, tacc) = d.put(q), d.put(a), d.put(acc)
    ctx.check(lib.h2b_flex_gate_fold_dev(ctx.h, pq, pa, hp(y), k, ext_k, pacc))
    assert np.array_equal(d.get(tacc), host.reshape(-1))


def test_quotient_folds_and_vanishing_division(env):
    """quotient_graph, permutation_fold, lookup_fold and divide_by_vanishing_poly, host columns against device columns"""
    from halo2_lib_b200 import evaluation as ev
    ctx, lib, _ = env
    d = Dev(env)
    k, ext_k, bf = 4, 6, 3
    n = 1 << ext_k
    host = [fr(100 + i, n) for i in range(12)]
    dev = [d.put(h)[0].value for h in host]
    ch = fr(113, 4)
    kw = dict(beta=ch[0], gamma=ch[1], theta=ch[2], y=ch[3])
    g = ev.GraphEvaluator()
    adv = [("advice", 0, r) for r in range(4)]
    gate = g.add_gates([("product", ("fixed", 0, 0), ("sum", ("sum", adv[0], ("product", adv[1], adv[2])), ("negated", adv[3])))])
    g2 = ev.GraphEvaluator()
    lk = g2.add_lookup([("product", ("fixed", 0, 0), ("advice", 0, 0))], [("fixed", 1, 0)])
    acc0 = fr(114, n)
    acc_h = acc0.copy()
    pacc, tacc = d.put(acc0)
    bh = ev.BoundGraph(g, gate, fixed=[host[0]], advice=[host[1]], **kw)
    bd = ev.BoundGraph(g, gate, fixed=[dev[0]], advice=[dev[1]], **kw)
    ctx.check(lib.h2b_quotient_graph(ctx.h, C.byref(bh.struct), k, ext_k, hp(acc_h)))
    ctx.check(lib.h2b_quotient_graph_dev(ctx.h, C.byref(bd.struct), k, ext_k, pacc))
    assert np.array_equal(d.get(tacc), acc_h.reshape(-1))
    hz, hc, hs = _ptrs(host[2:4]), _ptrs([host[1], host[4], host[5]]), _ptrs(host[6:9])
    tz, tc, ts = ((C.c_void_p * len(x))(*x) for x in (dev[2:4], [dev[1], dev[4], dev[5]], dev[6:9]))
    ctx.check(lib.h2b_permutation_fold(ctx.h, hz, 2, hc, hs, 3, 2, hp(host[9]), hp(host[10]), hp(host[11]), hp(ch[0]), hp(ch[1]),
                                       hp(ch[3]), bf, k, ext_k, hp(acc_h)))
    ctx.check(lib.h2b_permutation_fold_dev(ctx.h, tz, 2, tc, ts, 3, 2, vp(dev[9]), vp(dev[10]), vp(dev[11]), hp(ch[0]), hp(ch[1]),
                                           hp(ch[3]), bf, k, ext_k, pacc))
    assert np.array_equal(d.get(tacc), acc_h.reshape(-1))
    blh = ev.BoundGraph(g2, lk, fixed=[host[0], host[5]], advice=[host[1]], **kw)
    bld = ev.BoundGraph(g2, lk, fixed=[dev[0], dev[5]], advice=[dev[1]], **kw)
    ctx.check(lib.h2b_lookup_fold(ctx.h, C.byref(blh.struct), hp(host[2]), hp(host[4]), hp(host[6]), hp(host[9]), hp(host[10]),
                                  hp(host[11]), k, ext_k, hp(acc_h)))
    ctx.check(lib.h2b_lookup_fold_dev(ctx.h, C.byref(bld.struct), vp(dev[2]), vp(dev[4]), vp(dev[6]), vp(dev[9]), vp(dev[10]),
                                      vp(dev[11]), k, ext_k, pacc))
    assert np.array_equal(d.get(tacc), acc_h.reshape(-1))
    ctx.check(lib.h2b_divide_by_vanishing_poly(ctx.h, hp(acc_h), k, ext_k))
    ctx.check(lib.h2b_divide_by_vanishing_poly_dev(ctx.h, pacc, k, ext_k))
    assert np.array_equal(d.get(tacc), acc_h.reshape(-1))


def test_permute_expression_pair(env):
    ctx, lib, _ = env
    d = Dev(env)
    k, bf = 5, 5
    u = (1 << k) - bf - 1
    rng = np.random.default_rng(120)
    table = fr(121, u)
    inp = table[rng.integers(0, u, size=u)]
    outs = []
    for a in (inp, np.concatenate([inp[:-1], fr(122, 1)])):  # the second input misses the table
        hpi, hpt = np.empty_like(a), np.empty_like(a)
        rc_h = lib.h2b_permute_expression_pair(ctx.h, hp(a), hp(table), k, bf, hp(hpi), hp(hpt))
        (pa, _), (pt, _), (ppi, tpi), (ppt, tpt) = d.put(a), d.put(table), d.zeros(4 * u), d.zeros(4 * u)
        rc_d = lib.h2b_permute_expression_pair_dev(ctx.h, pa, pt, k, bf, ppi, ppt)
        outs.append((rc_h, rc_d))
        if rc_h == OK:
            assert np.array_equal(d.get(tpi), hpi.reshape(-1)) and np.array_equal(d.get(tpt), hpt.reshape(-1))
    assert outs == [(OK, OK), (UNSATISFIED, UNSATISFIED)]


# ------------------------------------------------------------------------------------------------ opening arithmetic
@pytest.mark.parametrize("n", [0, 1, 2, 500])
def test_opening_arithmetic(env, n):
    ctx, lib, _ = env
    d = Dev(env)
    a, z = fr(130 + n, n).reshape(-1, 4), fr(131, 1)[0]
    hv, dv = np.empty(4, dtype=np.uint64), np.empty(4, dtype=np.uint64)
    pa, _ = d.put(a)
    ctx.check(lib.h2b_eval_polynomial(ctx.h, hp(a), n, hp(z), hp(hv)))
    ctx.check(lib.h2b_eval_polynomial_dev(ctx.h, pa, n, hp(z), hp(dv)))
    assert np.array_equal(hv, dv)
    if n >= 1:
        hq = np.empty((max(n - 1, 1), 4), dtype=np.uint64)
        pq, tq = d.zeros(4 * max(n - 1, 1))
        ctx.check(lib.h2b_kate_division(ctx.h, hp(a), n, hp(z), hp(hq)))
        ctx.check(lib.h2b_kate_division_dev(ctx.h, pa, n, hp(z), pq))
        assert np.array_equal(d.get(tq, 4 * (n - 1)), hq.reshape(-1)[:4 * (n - 1)])
    polys, sc = [fr(132 + j, n).reshape(-1, 4) for j in range(3)], fr(135, 3)
    ho = np.empty((n, 4), dtype=np.uint64)
    ctx.check(lib.h2b_poly_lincomb(ctx.h, _ptrs(polys), hp(sc), 3, n, hp(ho)))
    dp = [d.put(p)[0] for p in polys]
    po, to = d.zeros(4 * n)
    ctx.check(lib.h2b_poly_lincomb_dev(ctx.h, (C.c_void_p * 3)(*[p.value if p else None for p in dp]), hp(sc), 3, n, po if n else None))
    assert np.array_equal(d.get(to, 4 * n), ho.reshape(-1))


# ------------------------------------------------------------------------------------------------ curve and SRS
@pytest.mark.parametrize("n", [0, 1, 37])
def test_curve_twins(env, n):
    """g1_fixed_base_mul, g1_sum, msm_g1_bases (n >= 1), check_on_curve, decompress"""
    ctx, lib, _ = env
    d = Dev(env)
    base = affine_to_limbs([pyref.G1])[0]
    sc = fr(140 + n, n).reshape(-1, 4)
    ho = np.empty((n, 8), dtype=np.uint64)
    ctx.check(lib.h2b_g1_fixed_base_mul(ctx.h, hp(base), hp(sc), n, hp(ho)))
    (ps, _), (po, to) = d.put(sc), d.zeros(8 * n)
    ctx.check(lib.h2b_g1_fixed_base_mul_dev(ctx.h, hp(base), ps if n else po, n, po))
    assert np.array_equal(d.get(to, 8 * n), ho.reshape(-1))
    pts = points(env, 141 + n, n) if n else np.zeros((0, 8), dtype=np.uint64)
    p3 = xyz(pts)
    hs = np.empty(12, dtype=np.uint64)
    ctx.check(lib.h2b_g1_sum(ctx.h, hp(p3), n, hp(hs)))
    (pp, _), (pso, tso) = d.put(p3), d.zeros(12)
    ctx.check(lib.h2b_g1_sum_dev(ctx.h, pp if n else pso, n, pso))
    assert np.array_equal(d.get(tso, 12), hs)
    if n:
        hm = np.empty(12, dtype=np.uint64)
        ctx.check(lib.h2b_msm_g1_bases(ctx.h, hp(pts), hp(sc), n, hp(hm)))
        (pb, _), (ps, _), (pmo, tmo) = d.put(pts), d.put(sc), d.zeros(12)
        ctx.check(lib.h2b_msm_g1_bases_dev(ctx.h, pb, ps, n, pmo))
        assert np.array_equal(d.get(tmo, 12), hm)
    bad = pts.copy()
    bad[::3, 4] ^= np.uint64(1)
    hc, dc = C.c_size_t(), C.c_size_t()
    ctx.check(lib.h2b_g1_check_on_curve(ctx.h, hp(bad), n, C.byref(hc)))
    pbad, _ = d.put(bad)
    ctx.check(lib.h2b_g1_check_on_curve_dev(ctx.h, pbad, n, C.byref(dc)))
    assert hc.value == dc.value == (n + 2) // 3
    pys = [pyref.g1_mul(3 + 11 * i, pyref.G1) for i in range(n)] + ([None] if n else [])
    blob = np.frombuffer(b"".join(pyref.g1_compress(p) for p in pys), dtype=np.uint8).copy()
    m = len(pys)
    hd, hi, di = np.empty((m, 8), dtype=np.uint64), C.c_size_t(7), C.c_size_t(7)
    ctx.check(lib.h2b_g1_decompress(ctx.h, hp(blob), m, hp(hd), C.byref(hi)))
    (pbl, _), (pdo, tdo) = d.put(blob.view(np.uint64) if m else np.zeros(0, dtype=np.uint64)), d.zeros(8 * m)
    ctx.check(lib.h2b_g1_decompress_dev(ctx.h, pbl, m, pdo if m else None, C.byref(di)))
    assert hi.value == di.value == 0
    assert np.array_equal(d.get(tdo, 8 * m), hd.reshape(-1))


@pytest.mark.parametrize("k", [0, 4])
def test_srs_utilities(env, k):
    """g_to_lagrange, srs_setup (both bases, then only one of them)"""
    ctx, lib, _ = env
    d = Dev(env)
    n = 1 << k
    base, tau = affine_to_limbs([pyref.G1])[0], fr(150 + k, 1)[0]
    hg, hgl = np.empty((n, 8), dtype=np.uint64), np.empty((n, 8), dtype=np.uint64)
    ctx.check(lib.h2b_srs_setup(ctx.h, hp(tau), hp(base), k, hp(hg), hp(hgl)))
    (pg, tg), (pgl, tgl) = d.zeros(8 * n), d.zeros(8 * n)
    ctx.check(lib.h2b_srs_setup_dev(ctx.h, hp(tau), hp(base), k, pg, pgl))
    assert np.array_equal(d.get(tg), hg.reshape(-1)) and np.array_equal(d.get(tgl), hgl.reshape(-1))
    only = np.empty((n, 8), dtype=np.uint64)
    ctx.check(lib.h2b_srs_setup(ctx.h, hp(tau), hp(base), k, None, hp(only)))
    assert np.array_equal(only, hgl)
    pts = points(env, 151 + k, n)
    hl = np.empty((n, 8), dtype=np.uint64)
    ctx.check(lib.h2b_g_to_lagrange(ctx.h, hp(pts), k, hp(hl)))
    (pp, _), (pl, tl) = d.put(pts), d.zeros(8 * n)
    ctx.check(lib.h2b_g_to_lagrange_dev(ctx.h, pp, k, pl))
    assert np.array_equal(d.get(tl), hl.reshape(-1))


def test_srs_upload_and_msm_twins(env):
    """handles from host and device bases commit alike; msm_g1 / _batch against msm_g1_dev / _batch_dev (the forms
    accumulate in different pipelines, so the commitments are compared normalised)"""
    ctx, lib, _ = env
    d = Dev(env)

    def norm(xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.uint64).reshape(-1, 12).copy()
        ctx.check(lib.h2b_g1_normalize(ctx.h, hp(xyz), len(xyz)))
        return xyz

    k = 6
    n = 1 << k
    g, gl = points(env, 160, n), points(env, 161, n)
    hh, hd = vp(), vp()
    ctx.check(lib.h2b_srs_upload(ctx.h, hp(g), hp(gl), k, 0, n, C.byref(hh)))
    (pg, _), (pgl, _) = d.put(g), d.put(gl)
    ctx.check(lib.h2b_srs_upload_dev(ctx.h, pg, pgl, k, 0, n, C.byref(hd)))
    try:
        cols = [fr(162 + j, n) for j in range(3)]
        basis = (C.c_int * 3)(0, 1, 1)
        hb = np.empty((3, 12), dtype=np.uint64)
        ctx.check(lib.h2b_msm_g1_batch(ctx.h, hh, basis, _ptrs(cols), 3, n, hp(hb)))
        dcols = [d.put(c)[0].value for c in cols]
        po, to = d.zeros(36)
        ctx.check(lib.h2b_msm_g1_batch_dev(ctx.h, hd, basis, (C.c_void_p * 3)(*dcols), 3, n, po))
        assert np.array_equal(norm(d.get(to)), norm(hb))
        for j, b in enumerate((0, 1, 1)):
            h1 = np.empty(12, dtype=np.uint64)
            ctx.check(lib.h2b_msm_g1(ctx.h, hh, b, hp(cols[j]), n, hp(h1)))
            p1, t1 = d.zeros(12)
            ctx.check(lib.h2b_msm_g1_dev(ctx.h, hd, b, vp(dcols[j]), n, p1))
            assert np.array_equal(norm(d.get(t1)), norm(h1)) and np.array_equal(norm(h1), norm(hb[j]))
    finally:
        lib.h2b_srs_destroy(ctx.h, hh)
        lib.h2b_srs_destroy(ctx.h, hd)


# ------------------------------------------------------------------------------------------------ bad arguments
def test_bad_arguments_keep_their_status_and_the_context(env):
    ctx, lib, _ = env
    d = Dev(env)
    a = fr(170, 64)
    w = np.zeros(4, dtype=np.uint64)
    out = np.empty((1 << 8, 8), dtype=np.uint64)
    pa, _ = d.put(a)
    h = ctx.h
    calls = {
        "ntt_fr null": lambda: lib.h2b_ntt_fr(h, None, 6, hp(w), 0),
        "ntt_fr_dev null": lambda: lib.h2b_ntt_fr_dev(h, None, 6, hp(w), 0),
        "ntt_fr null omega": lambda: lib.h2b_ntt_fr(h, hp(a), 6, None, 0),
        "ntt_fr_dev null omega": lambda: lib.h2b_ntt_fr_dev(h, pa, 6, None, 0),
        "ntt_fr log_n": lambda: lib.h2b_ntt_fr(h, hp(a), 29, hp(w), 0),
        "ntt_fr_dev log_n": lambda: lib.h2b_ntt_fr_dev(h, pa, 29, hp(w), 0),
        "lagrange_to_coeff k": lambda: lib.h2b_lagrange_to_coeff(h, hp(a), 29),
        "lagrange_to_coeff_dev k": lambda: lib.h2b_lagrange_to_coeff_dev(h, pa, 29),
        "extended_to_coeff null": lambda: lib.h2b_extended_to_coeff(h, None, 6),
        "coeff_to_extended ext_k": lambda: lib.h2b_coeff_to_extended(h, hp(a), 64, 29, hp(out)),
        "coeff_to_extended n_coeffs": lambda: lib.h2b_coeff_to_extended(h, hp(a), 64, 5, hp(out)),
        "coeff_to_extended_dev n_coeffs": lambda: lib.h2b_coeff_to_extended_dev(h, pa, 64, 5, pa),
        "lagrange_to_coeff_batch k": lambda: lib.h2b_lagrange_to_coeff_batch(h, _ptrs([a]), 1, 29),
        "coeff_to_lagrange_batch null": lambda: lib.h2b_coeff_to_lagrange_batch(h, None, 1, 6),
        "coeff_to_lagrange_batch null column": lambda: lib.h2b_coeff_to_lagrange_batch(h, (C.c_void_p * 1)(None), 1, 6),
        "coeff_to_extended_batch n_coeffs": lambda: lib.h2b_coeff_to_extended_batch(h, _ptrs([a]), 1, 64, 5, _ptrs([out])),
        "fused batch ext_k < k": lambda: lib.h2b_lagrange_to_coeff_and_extended_batch(h, _ptrs([a]), 1, 6, 5, _ptrs([out])),
        "fused batch ext_k": lambda: lib.h2b_lagrange_to_coeff_and_extended_batch(h, _ptrs([a]), 1, 6, 29, _ptrs([out])),
        "assign_columns k": lambda: lib.h2b_assign_columns(h, hp(a), 16, None, 0, 29, 1, hp(out)),
        "assign_columns_dev k": lambda: lib.h2b_assign_columns_dev(h, pa, 16, None, 0, 29, 1, pa),
        "assign_columns null": lambda: lib.h2b_assign_columns(h, None, 16, None, 0, 4, 1, hp(out)),
        "assign_columns_assigned k": lambda: lib.h2b_assign_columns_assigned(h, hp(a), 4, None, 0, 29, 1, hp(out)),
        "assign_lookups k": lambda: lib.h2b_assign_lookups(h, hp(a), 16, 29, 1, hp(out)),
        "assign_lookups_dev k": lambda: lib.h2b_assign_lookups_dev(h, pa, 16, 29, 1, pa),
        "eval_rational null": lambda: lib.h2b_eval_rational(h, None, hp(a), 4, hp(out)),
        "batch_invert null": lambda: lib.h2b_batch_invert_fr(h, None, 4),
        "grand_product null start": lambda: lib.h2b_grand_product_fr(h, hp(a), None, 4, hp(out)),
        "flex_gate ext_k": lambda: lib.h2b_flex_gate_fold(h, hp(a), hp(a), hp(w), 4, 29, hp(out)),
        "flex_gate ext_k < k": lambda: lib.h2b_flex_gate_fold(h, hp(a), hp(a), hp(w), 6, 5, hp(out)),
        "flex_gate_dev ext_k < k": lambda: lib.h2b_flex_gate_fold_dev(h, pa, pa, hp(w), 6, 5, pa),
        "divide_by_vanishing ext_k == k": lambda: lib.h2b_divide_by_vanishing_poly(h, hp(a), 6, 6),
        "divide_by_vanishing_dev ext_k == k": lambda: lib.h2b_divide_by_vanishing_poly_dev(h, pa, 6, 6),
        "divide_by_vanishing ext_k": lambda: lib.h2b_divide_by_vanishing_poly(h, hp(a), 4, 29),
        "g_to_lagrange k": lambda: lib.h2b_g_to_lagrange(h, hp(out), 29, hp(out)),
        "g_to_lagrange_dev k": lambda: lib.h2b_g_to_lagrange_dev(h, pa, 29, pa),
        "srs_setup k": lambda: lib.h2b_srs_setup(h, hp(w), hp(w), 29, hp(out), None),
        "srs_setup_dev k": lambda: lib.h2b_srs_setup_dev(h, hp(w), hp(w), 29, pa, None),
        "srs_upload k": lambda: lib.h2b_srs_upload(h, hp(out), None, 28, 0, 4, C.byref(vp())),
        "srs_upload null handle": lambda: lib.h2b_srs_upload(h, hp(out), None, 2, 0, 4, None),
        "srs_upload_dev k": lambda: lib.h2b_srs_upload_dev(h, pa, None, 28, 0, 4, C.byref(vp())),
        "check_on_curve null": lambda: lib.h2b_g1_check_on_curve(h, hp(out), 4, None),
        "decompress null": lambda: lib.h2b_g1_decompress(h, hp(out), 4, hp(out), None),
        "permute_expression_pair k": lambda: lib.h2b_permute_expression_pair(h, hp(a), hp(a), 29, 5, hp(out), hp(out)),
        "permute_expression_pair no rows": lambda: lib.h2b_permute_expression_pair(h, hp(a), hp(a), 2, 3, hp(out), hp(out)),
        "quotient_graph null": lambda: lib.h2b_quotient_graph(h, None, 4, 6, hp(out)),
        "lookup_fold null": lambda: lib.h2b_lookup_fold(h, None, hp(a), hp(a), hp(a), hp(a), hp(a), hp(a), 4, 6, hp(out)),
        "permutation_fold null": lambda: lib.h2b_permutation_fold(h, None, 1, None, None, 1, 1, None, None, None, hp(w), hp(w), hp(w),
                                                                  3, 4, 6, hp(out)),
        "eval_polynomial null": lambda: lib.h2b_eval_polynomial(h, None, 4, hp(w), hp(w)),
        "kate_division empty": lambda: lib.h2b_kate_division(h, hp(a), 0, hp(w), hp(out)),
        "kate_division_dev empty": lambda: lib.h2b_kate_division_dev(h, pa, 0, hp(w), vp(int(pa.value) + 1024)),
        "poly_lincomb m = 0": lambda: lib.h2b_poly_lincomb(h, _ptrs([a]), hp(w), 0, 4, hp(out)),
        "poly_lincomb m = 33": lambda: lib.h2b_poly_lincomb(h, _ptrs([a] * 33), hp(a), 33, 4, hp(out)),
        "poly_lincomb_dev m = 33": lambda: lib.h2b_poly_lincomb_dev(h, (C.c_void_p * 33)(*[pa.value] * 33), hp(a), 33, 4, pa),
        "msm_g1_bases n = 0": lambda: lib.h2b_msm_g1_bases(h, hp(out), hp(a), 0, hp(out)),
        "msm_g1_bases_dev n = 0": lambda: lib.h2b_msm_g1_bases_dev(h, pa, pa, 0, pa),
        "g1_sum null": lambda: lib.h2b_g1_sum(h, None, 4, hp(out)),
        "g1_fixed_base_mul null": lambda: lib.h2b_g1_fixed_base_mul(h, hp(w), None, 4, hp(out)),
    }
    got, msgs = {}, {}
    for name, call in calls.items():
        got[name] = call()
        msgs[name] = lib.h2b_last_error(h).decode()
    assert got == {name: ARG for name in calls}
    # the message of each failure, where the host form and its `_dev` twin test the same condition with the same words
    want = {
        "ntt_fr log_n": "ntt: log_n exceeds the two-adicity of Fr (28)",
        "ntt_fr_dev log_n": "ntt: log_n exceeds the two-adicity of Fr (28)",
        "lagrange_to_coeff k": "ntt: log_n exceeds the two-adicity of Fr (28)",
        "lagrange_to_coeff_dev k": "ntt: log_n exceeds the two-adicity of Fr (28)",
        "coeff_to_extended n_coeffs": "coeff_to_extended: sizes out of range",
        "coeff_to_extended_dev n_coeffs": "coeff_to_extended: sizes out of range",
        "lagrange_to_coeff_batch k": "ntt batch: sizes out of range",
        "coeff_to_lagrange_batch null column": "ntt batch: null column",
        "fused batch ext_k < k": "ntt batch: sizes out of range",
        "assign_columns k": "assign: k out of range",
        "assign_columns_dev k": "assign: k out of range",
        "assign_lookups k": "assign: k out of range",
        "assign_lookups_dev k": "assign: k out of range",
        "flex_gate ext_k < k": "flex_gate: extended_k out of range",
        "flex_gate_dev ext_k < k": "flex_gate: extended_k out of range",
        "g_to_lagrange k": "g_to_lagrange: k out of range",
        "g_to_lagrange_dev k": "g_to_lagrange: k out of range",
        "srs_setup k": "srs_setup: k out of range",
        "srs_setup_dev k": "srs_setup: k out of range",
        "srs_upload k": "srs: bad shard",
        "permute_expression_pair k": "permute_expression_pair: no usable rows",
        "quotient_graph null": "quotient_graph: null pointer",
        "kate_division empty": "kate_division: empty polynomial",
        "kate_division_dev empty": "kate_division: empty polynomial",
        "poly_lincomb m = 33": "poly_lincomb: 1..32 polynomials per call",
        "poly_lincomb_dev m = 33": "poly_lincomb: 1..32 polynomials per call",
        "msm_g1_bases n = 0": "msm: null pointer or n == 0",
        "msm_g1_bases_dev n = 0": "msm: null pointer or n == 0",
    }
    assert {name: msgs[name] for name in want} == want
    # the context still works
    x = fr(171, 8)
    want = x.copy()
    ctx.check(lib.h2b_batch_invert_fr(h, hp(want), 8))
    px, tx = d.put(x)
    ctx.check(lib.h2b_batch_invert_fr_dev(h, px, 8))
    assert np.array_equal(d.get(tx), want.reshape(-1))


def test_ctx_create_multi_failures_leave_no_context(env):
    """a duplicate device id and a device that does not exist fail with H2B_ERR_ARG and their message; the contexts made
    before the failure are destroyed, and a one-device group works like a plain context"""
    ctx, lib, _ = env
    for ids, msg in (([0, 0], "ctx_create_multi: duplicate device id"), ([0, 1 << 20], "device index out of range")):
        out = vp(12345)
        arr = (C.c_int * len(ids))(*ids)
        assert lib.h2b_ctx_create_multi(arr, len(ids), C.byref(out)) == ARG
        assert out.value is None and lib.h2b_last_error(None).decode() == msg
    out = vp()
    assert lib.h2b_ctx_create(-1, C.byref(out)) == ARG and out.value is None
    assert lib.h2b_last_error(None).decode() == "device index out of range"
    assert lib.h2b_ctx_create_multi((C.c_int * 1)(0), 1, C.byref(out)) == OK
    try:
        assert lib.h2b_ctx_device_count(out) == 1
        x = fr(180, 8)
        want, got = x.copy(), x.copy()
        ctx.check(lib.h2b_batch_invert_fr(ctx.h, hp(want), 8))
        assert lib.h2b_batch_invert_fr(out, hp(got), 8) == OK
        assert np.array_equal(got, want)
    finally:
        lib.h2b_ctx_destroy(out)
