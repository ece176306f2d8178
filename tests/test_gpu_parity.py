"""GPU parity tests (-m gpu): every call goes through the C ABI of libh2b200.so (ctypes) and is compared
bit-exactly with the CPU oracle (oracle/) on the same seeded inputs.  Integer arithmetic: the bar is equality."""
import numpy as np
import pytest
from oracle import pyref, oracle as orc
from util import *

pytestmark = pytest.mark.gpu
P, R = pyref.P, pyref.R


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


# ------------------------------------------------------------------ L0: field arithmetic of the kernels
@pytest.mark.parametrize("which,m", [(0, P), (1, R)], ids=["Fq", "Fr"])
def test_field_ops(ctx, h2b, which, m):
    rng = np.random.default_rng(100 + which)
    edge = [0, 1, 2, m - 1, m - 2, (1 << 64) - 1, 1 << 64, (1 << 128) - 1, 1 << 253, m >> 1, (1 << 32) - 1, 1 << 32]
    a = edge + rand_ints(rng, 4000, m)
    b = list(reversed(edge)) + rand_ints(rng, 4000, m)
    A, B = mont(a, m), mont(b, m)
    assert np.array_equal(ctx.field_op(which, 0, A, B), orc.f_mul(which, A, B))
    assert np.array_equal(ctx.field_op(which, 1, A, B), orc.f_add(which, A, B))
    assert np.array_equal(ctx.field_op(which, 2, A, B), orc.f_sub(which, A, B))
    assert np.array_equal(ctx.field_op(which, 4, A), orc.from_mont(which, A))
    assert np.array_equal(ctx.field_op(which, 6, A), orc.f_mul(which, A, A))  # dedicated squaring
    assert np.array_equal(ctx.field_op(which, 6, B), orc.f_mul(which, B, B))
    # fused two-product routine of the group law: a*b + (a+b)(a-b) and a*b - b*b
    sm, df = orc.f_add(which, A, B), orc.f_sub(which, A, B)
    assert np.array_equal(ctx.field_op(which, 7, A, B), orc.f_add(which, orc.f_mul(which, A, B), orc.f_mul(which, sm, df)))
    assert np.array_equal(ctx.field_op(which, 8, A, B), orc.f_sub(which, orc.f_mul(which, A, B), orc.f_mul(which, B, B)))
    ea2 = mont([x for x in edge for _ in edge], m)
    eb2 = mont([y for _ in edge for y in edge], m)
    assert np.array_equal(ctx.field_op(which, 8, ea2, eb2), orc.f_sub(which, orc.f_mul(which, ea2, eb2), orc.f_mul(which, eb2, eb2)))
    assert np.array_equal(ctx.field_op(which, 5, ints_to_limbs(a)), A)
    assert np.array_equal(ctx.field_op(which, 3, A[:300]), orc.f_inv(which, A[:300]))
    assert np.array_equal(ctx.field_op(which, 9, A[:600]), orc.f_inv(which, A[:600]))  # binary-Euclid inversion (single-lane paths)
    with pytest.raises(h2b.H2BError):  # the ops end at 10
        ctx.field_op(which, 11, A[:3000])
    # products of edge x edge (carry patterns)
    ea = [x for x in edge for _ in edge]
    eb = [y for _ in edge for y in edge]
    assert unmont(ctx.field_op(which, 0, mont(ea, m), mont(eb, m)), m) == [x * y % m for x, y in zip(ea, eb)]


# ------------------------------------------------------------------ group helpers
def test_fixed_base_mul_and_sum(ctx):
    rng = np.random.default_rng(7)
    sc = [0, 1, 2, R - 1, 12345] + rand_ints(rng, 60, R)
    g = affine_to_limbs([pyref.G1])[0]
    got = ctx.g1_fixed_base_mul(g, mont(sc, R))
    want = orc.g1_fixed_base_mul(mont(sc, R), g)
    assert np.array_equal(got, want)
    assert jac_limbs_to_affine(np.concatenate([got[4], mont([1], P)[0]])) == pyref.g1_mul(12345, pyref.G1)
    # g1_sum over Jacobian points incl. identity and P + (-P)
    pts = [orc.g1_scalar_mul(mont([s], R)[0], g) for s in (5, 7, R - 5, 0, 9)]
    s = norm(ctx, ctx.g1_sum(np.stack(pts)))
    assert jac_limbs_to_affine(s) == pyref.g1_mul(16, pyref.G1)
    assert jac_limbs_to_affine(norm(ctx, ctx.g1_sum(np.stack([pts[0], pts[2]])))) is None
    assert jac_limbs_to_affine(norm(ctx, ctx.g1_sum(np.stack([pts[0], pts[0]])))) == pyref.g1_mul(10, pyref.G1)


def test_eip196_public_vectors_on_the_gpu(ctx, h2b):
    """the public EIP-196 ecMul / ecAdd vectors (tests/golden/eip196_vectors.json) through the CUDA group law: fixed-base
    multiplication, the ad-hoc MSM (n = 1, 2) and g1_sum"""
    import json, os
    v = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "eip196_vectors.json")))
    pt = lambda x, y: None if (int(x, 16) == 0 and int(y, 16) == 0) else (int(x, 16), int(y, 16))
    for e in v["ecmul"]:
        p, want, s = pt(e["x"], e["y"]), pt(e["rx"], e["ry"]), int(e["scalar"], 16) % R
        base = affine_to_limbs([p])
        got = ctx.g1_fixed_base_mul(base[0], mont([s], R))[0]
        assert np.array_equal(got, affine_to_limbs([want])[0]), e["name"]
        out = norm(ctx, h2b.best_multiexp(ctx, mont([s], R), base))
        assert jac_limbs_to_affine(out) == want, e["name"]
    for e in v["ecadd"]:
        a, b, want = pt(e["x1"], e["y1"]), pt(e["x2"], e["y2"]), pt(e["rx"], e["ry"])
        out = norm(ctx, h2b.best_multiexp(ctx, mont([1, 1], R), affine_to_limbs([a, b])))
        assert jac_limbs_to_affine(out) == want, e["name"]
        jac = np.zeros((2, 12), dtype=np.uint64)
        for i, q in enumerate((a, b)):
            if q is None:
                jac[i, 4:8] = mont([1], P)[0]
            else:
                jac[i, :8] = affine_to_limbs([q])[0]
                jac[i, 8:] = mont([1], P)[0]
        assert jac_limbs_to_affine(norm(ctx, ctx.g1_sum(jac))) == want, e["name"]


# ------------------------------------------------------------------ L1: MSM
def _bases(ctx, n, a0=3, delta=5):
    """b_i = (a0 + i*delta) * G built on the GPU (itself checked against the oracle above)."""
    g = affine_to_limbs([pyref.G1])[0]
    sc = mont([a0 + i * delta for i in range(n)], R)
    return ctx.g1_fixed_base_mul(g, sc)


def test_msm_adhoc_small_vs_naive(ctx, h2b):
    rng = np.random.default_rng(11)
    n = 100
    B = _bases(ctx, n)
    B[7] = 0  # identity base (halo2-ecc/src/ecc/pippenger.rs:216-218)
    B[9] = B[8]  # repeated base
    sc = rand_ints(rng, n, R)
    sc[0], sc[1], sc[2] = 0, 1, R - 1  # halo2-ecc/src/secp256k1/tests/mod.rs:87-109
    S = mont(sc, R)
    got = norm(ctx, h2b.best_multiexp(ctx, S, B))
    assert np.array_equal(got, orc.msm_naive(S, B))


def test_msm_edge_cases(ctx, h2b):
    g11 = _bases(ctx, 1, a0=11)[0]
    B2 = np.stack([g11, g11])
    # sums to infinity (halo2-ecc/src/bn254/tests/msm_sum_infinity.rs:16-69)
    out = norm(ctx, h2b.best_multiexp(ctx, mont([5, R - 5], R), B2))
    assert np.array_equal(out, orc.msm_naive(mont([5, R - 5], R), B2))
    assert jac_limbs_to_affine(out) is None
    # all-zero scalars (keygen-style column, halo2-base/benches/inner_product.rs:41)
    B = _bases(ctx, 64)
    out = norm(ctx, h2b.best_multiexp(ctx, np.zeros((64, 4), dtype=np.uint64), B))
    assert jac_limbs_to_affine(out) is None
    # n = 1 and all-equal scalars with equal bases (doubling path inside buckets)
    out = norm(ctx, h2b.best_multiexp(ctx, mont([R - 1], R), B[:1]))
    assert np.array_equal(out, orc.msm_naive(mont([R - 1], R), B[:1]))
    Beq = np.repeat(B[:1], 300, axis=0)
    Seq = mont([123456789] * 300, R)
    assert np.array_equal(norm(ctx, h2b.best_multiexp(ctx, Seq, Beq)), orc.msm_pippenger(Seq, Beq))


@pytest.mark.parametrize("k,dist", [(6, "uniform"), (10, "uniform"), (10, "witness"), (13, "witness"), (14, "uniform")])
def test_msm_srs_vs_pippenger(ctx, h2b, k, dist):
    n = 1 << k
    rng = np.random.default_rng(0xB2000000 + k)
    B = _bases(ctx, n, a0=1 + k, delta=7)
    sc = rand_ints(rng, n, R) if dist == "uniform" else witness_like_ints(rng, n)
    S = mont(sc, R)
    params = h2b.ParamsKZG(ctx, k, g=B, g_lagrange=B[::-1].copy())
    want = orc.msm_pippenger(S, B)
    assert np.array_equal(norm(ctx, params.commit(S)), want)
    assert np.array_equal(norm(ctx, params.commit_lagrange(S)), orc.msm_pippenger(S, B[::-1].copy()))
    # ad-hoc path on the same input
    assert np.array_equal(norm(ctx, h2b.best_multiexp(ctx, S, B)), want)
    # batch API: three columns, same basis
    S2 = mont(witness_like_ints(rng, n), R)
    outs = params.commit_batch(0, [S, S2, S])
    assert np.array_equal(norm(ctx, outs[0]), want) and np.array_equal(norm(ctx, outs[2]), want)
    assert np.array_equal(norm(ctx, outs[1]), orc.msm_pippenger(S2, B))
    params.close()


def test_msm_hot_bucket_and_sharded(ctx, h2b):
    # one scalar value repeated for most of the column: a single bucket spans thousands of chunks (big-bucket path)
    k = 13
    n = 1 << k
    rng = np.random.default_rng(5)
    B = _bases(ctx, n, a0=2, delta=3)
    sc = [1] * (n - 100) + rand_ints(rng, 100, R)
    S = mont(sc, R)
    want = orc.msm_pippenger(S, B)
    params = h2b.ParamsKZG(ctx, k, g=B)
    assert np.array_equal(norm(ctx, params.commit(S)), want)
    params.close()
    # point-range sharding as on G GPUs: partial sums over [g*n/G, (g+1)*n/G) then g1_sum == full MSM
    G = 4
    parts = []
    for g in range(G):
        p = h2b.ParamsKZG(ctx, k, g=B, begin=g * n // G, count=n // G)
        parts.append(p.commit(S[g * n // G:(g + 1) * n // G]))
        p.close()
    assert np.array_equal(norm(ctx, ctx.g1_sum(np.stack(parts))), want)


def test_msm_odd_shard_and_long_batch(ctx, h2b):
    """a shard that is not a power of two (begin/count arbitrary) and a batch longer than twice the number of lanes"""
    k = 10
    n = 1 << k
    rng = np.random.default_rng(77)
    B = _bases(ctx, n, a0=9, delta=4)
    begin, count = 100, 777
    p = h2b.ParamsKZG(ctx, k, g=B, g_lagrange=B, begin=begin, count=count)
    cols = [mont(rand_ints(rng, count, R) if j % 2 == 0 else witness_like_ints(rng, count), R) for j in range(7)]
    outs = p.commit_batch([j % 2 for j in range(7)], cols)
    for j in range(7):
        assert np.array_equal(norm(ctx, outs[j]), orc.msm_pippenger(cols[j], B[begin:begin + count]))
    # wrong length is rejected, not mis-indexed
    with pytest.raises(h2b.H2BError):
        p.commit(cols[0][:-1])
    p.close()


def test_msm_closed_form_large(ctx, h2b):
    # size-independent property at 2^17: bases a_i*G (a_i = a0 + i*delta) => MSM == (sum s_i a_i mod r)*G
    k = 17
    n = 1 << k
    rng = np.random.default_rng(0xB2000000 + k)
    a0, delta = 987654321, 123456789
    B = _bases(ctx, n, a0=a0, delta=delta)
    sc = rand_ints(rng, n // 2, R) + witness_like_ints(rng, n // 2)
    S = mont(sc, R)
    params = h2b.ParamsKZG(ctx, k, g=B)
    got = jac_limbs_to_affine(norm(ctx, params.commit(S)))
    kk = sum(s * (a0 + i * delta) for i, s in enumerate(sc)) % R
    assert got == pyref.g1_mul(kk, pyref.G1)
    # linearity: commit(S) + commit(S) == commit(2S)
    S2 = mont([2 * s % R for s in sc], R)
    two = norm(ctx, ctx.g1_sum(np.stack([params.commit(S), params.commit(S)])))
    assert np.array_equal(two, norm(ctx, params.commit(S2)))
    params.close()


@pytest.mark.parametrize("group", [0, 1, 2, 3, 5, 16])
def test_msm_group_pipeline(h2b, group):
    """option "msm.batch_group": the MSMs of one batch call share ONE sort / accumulate / bucket-reduction pipeline (bucket
    sets side by side, sorted entries carry the table bit).  Whatever the grouping, every commitment is the oracle's: two
    distinct bases mixed inside a group, an all-zero column, a hot-bucket column, witness-like and uniform columns, batches
    longer than a group and longer than groups x lanes — through the device-pointer and the host-pointer batch calls."""
    import torch
    c = h2b.Context(0)
    c.set_option("msm.batch_group", group)
    try:
        rng = np.random.default_rng(4242 + group)
        for k, m in [(9, 13), (12, 7), (6, 35)]:
            n = 1 << k
            Bm = _bases(c, n, a0=3 + k, delta=5)
            Bl = _bases(c, n, a0=1000 + k, delta=7)
            Bl[2] = 0  # identity base in one of the two tables
            cols = []
            for j in range(m):
                if j == 1:
                    sc = [0] * n
                elif j == 2:
                    sc = [1] * (n - 9) + rand_ints(rng, 9, R)
                elif j % 3 == 0:
                    sc = witness_like_ints(rng, n)
                else:
                    sc = rand_ints(rng, n, R)
                cols.append(mont(sc, R))
            basis = [(j * 7 // 3) % 2 for j in range(m)]
            want = [orc.msm_pippenger(cols[j], Bl if basis[j] else Bm) for j in range(m)]
            params = h2b.ParamsKZG(c, k, g=Bm, g_lagrange=Bl)
            outs = params.commit_batch(basis, cols)  # host pointers
            for j in range(m):
                assert np.array_equal(norm(c, outs[j]), want[j]), (k, j, "host")
            d_cols = [torch.from_numpy(x.view(np.int64)).cuda() for x in cols]
            d_out = torch.zeros((m, 12), dtype=torch.int64, device="cuda")
            params.commit_batch_dev(basis, [t.data_ptr() for t in d_cols], n, d_out.data_ptr())
            torch.cuda.synchronize()
            outs = d_out.cpu().numpy().view(np.uint64)
            for j in range(m):
                assert np.array_equal(norm(c, outs[j]), want[j]), (k, j, "dev")
            params.close()
        with pytest.raises(h2b.H2BError):
            c.set_option("msm.batch_group", 17)
    finally:
        c.close()


@pytest.mark.parametrize("k,case", [(6, "uniform"), (10, "witness"), (13, "uniform"), (13, "zero"), (9, "one-base")])
def test_msm_table_edge_vectors(ctx, h2b, k, case):
    """the tabulated-SRS MSM (ParamsKZG.commit) on the inputs that stress the bucket accumulation: identity bases, repeated
    bases (P + P inside a bucket), P + (-P) cancelling inside a bucket, an all-zero column, and one base repeated 512 times
    with one repeated scalar (every entry in one bucket)."""
    n = 1 << k
    rng = np.random.default_rng(900 + k)
    if case == "one-base":
        B = np.repeat(_bases(ctx, 1, a0=2, delta=3), n, axis=0)
        S = mont([123456789] * n, R)
    elif case == "zero":
        B = _bases(ctx, n, a0=2, delta=3)
        S = np.zeros((n, 4), dtype=np.uint64)
    else:
        B = _bases(ctx, n, a0=5 + k, delta=3)
        B[3] = 0            # identity base (0,0)
        B[11] = B[10]       # repeated base: equal points meet in one bucket
        sc = rand_ints(rng, n, R) if case == "uniform" else witness_like_ints(rng, n)
        sc[10], sc[11] = 777, 777                      # P + P inside a bucket
        sc[20], sc[21] = 424242, 424242
        B[21, 4:] = mont([(P - v) % P for v in unmont(B[20, 4:].reshape(1, 4), P)], P)[0]  # B[21] = -B[20]: cancels
        B[21, :4] = B[20, :4]
        S = mont(sc, R)
    params = h2b.ParamsKZG(ctx, k, g=B)
    try:
        got = norm(ctx, params.commit(S))
    finally:
        params.close()
    assert np.array_equal(got, orc.msm_pippenger(S, B)), (k, case)
    if case == "zero":
        assert jac_limbs_to_affine(got) is None


def test_set_option_rejects_unknown_keys(h2b):
    """a key that is not one of the switches listed in include/h2b200.h fails with H2BError instead of being ignored"""
    c = h2b.Context(0)
    try:
        for key in ("msm.affine_levels", "msm.affine_k", "msm.affine_per_thread_inverse", "msm.tail_priority", "no.such.option"):
            with pytest.raises(h2b.H2BError):
                c.set_option(key, 1)
    finally:
        c.close()


# ------------------------------------------------------------------ L2: NTT
@pytest.mark.parametrize("k", [0, 1, 2, 3, 5, 8, 10, 11, 12, 13, 16, 20, 21])
def test_ntt_vs_oracle(ctx, h2b, k):
    rng = np.random.default_rng(0xB2001000 + k)
    n = 1 << k
    raw = rng.integers(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    raw[:, 3] &= np.uint64((1 << 60) - 1)  # < r: valid Montgomery residues
    A = raw
    w = orc.omega(k)
    assert np.array_equal(h2b.omega(k), w)
    got = h2b.best_fft(ctx, A, w, k)
    assert np.array_equal(got, orc.ntt(A, k, w))
    dom = h2b.EvaluationDomain(ctx, 3, k)
    assert np.array_equal(dom.lagrange_to_coeff(got), A)
    assert np.array_equal(dom.coeff_to_lagrange(A), got)
    if k <= 8:  # definition check against the O(n^2) DFT
        a = unmont(A, R)
        assert unmont(got, R) == pyref.dft(a, pyref.omega_for(k))


@pytest.mark.parametrize("k,j", [(3, 3), (5, 4), (8, 5), (12, 5), (14, 4), (17, 5)])
def test_coset_extended(ctx, h2b, k, j):
    rng = np.random.default_rng(0xB2001000 + 100 + k)
    n = 1 << k
    A = mont(rand_ints(rng, n, R), R) if k <= 12 else None
    if A is None:
        raw = rng.integers(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
        raw[:, 3] &= np.uint64((1 << 60) - 1)
        A = raw
    dom = h2b.EvaluationDomain(ctx, j, k)
    assert dom.extended_k == k + {3: 1, 4: 2, 5: 2}[j]
    ext = dom.coeff_to_extended(A)
    assert np.array_equal(ext, orc.coeff_to_extended(A, dom.extended_k))
    back = dom.extended_to_coeff(ext)
    full = orc.extended_to_coeff(ext, dom.extended_k)
    assert np.array_equal(back, full[: n * (j - 1)])
    assert np.array_equal(back[:n], A) and not back[n:].any()


def test_ntt_batch_pipelined(ctx, h2b):
    k = 12
    rng = np.random.default_rng(5150)
    cols = [mont(rand_ints(rng, 1 << k, R), R) for _ in range(7)]
    dom = h2b.EvaluationDomain(ctx, 5, k)
    coeffs = dom.lagrange_to_coeff_many(cols)
    exts = dom.coeff_to_extended_many(coeffs)
    for c, co, ex in zip(cols, coeffs, exts):
        assert np.array_equal(co, orc.lagrange_to_coeff(c, k))
        assert np.array_equal(ex, orc.coeff_to_extended(co, dom.extended_k))
    # the fused call (coefficients stay on the device between the two transforms) gives the same pair of results
    for m in (1, 2, 7):
        co2, ex2 = dom.lagrange_to_coeff_and_extended_many(cols[:m])
        for j in range(m):
            assert np.array_equal(co2[j], coeffs[j]) and np.array_equal(ex2[j], exts[j])


# ------------------------------------------------------------------ L3: KZG identity ties MSM, NTT and SRS layout together
def test_kzg_commit_identity(ctx, h2b):
    k = 10
    n = 1 << k
    rng = np.random.default_rng(33)
    tau = rand_ints(rng, 1, R)[0]
    g = affine_to_limbs([pyref.G1])[0]
    w = pyref.omega_for(k)
    mono = [pow(tau, i, R) for i in range(n)]
    # L_i(tau) = (tau^n - 1) * w^i / (n * (tau - w^i))
    tn = (pow(tau, n, R) - 1) % R
    ninv = pow(n, -1, R)
    lag = [tn * pow(w, i, R) % R * ninv % R * pow((tau - pow(w, i, R)) % R, -1, R) % R for i in range(n)]
    G = ctx.g1_fixed_base_mul(g, mont(mono, R))
    GL = ctx.g1_fixed_base_mul(g, mont(lag, R))
    params = h2b.ParamsKZG(ctx, k, g=G, g_lagrange=GL)
    evals = rand_ints(rng, n, R)
    E = mont(evals, R)
    dom = h2b.EvaluationDomain(ctx, 4, k)
    coeffs = dom.lagrange_to_coeff(E)
    c1 = norm(ctx, params.commit_lagrange(E))
    c2 = norm(ctx, params.commit(coeffs))
    assert np.array_equal(c1, c2)
    p_tau = sum(c * pow(tau, i, R) for i, c in enumerate(unmont(coeffs, R))) % R
    assert jac_limbs_to_affine(c1) == pyref.g1_mul(p_tau, pyref.G1)
    params.close()


# ------------------------------------------------------------------ witness assignment
def test_assign_witnesses_vs_oracle(ctx, h2b):
    rng = np.random.default_rng(30)
    k, ncols, min_rows = 8, 5, 9
    max_rows = (1 << k) - min_rows
    threads, sels, total = [], [], 0
    while total < 4 * max_rows - 50:
        ln = int(rng.integers(0, 90))
        threads.append(mont([int(v) for v in rng.integers(0, 1 << 62, size=ln)], R) if ln else np.zeros((0, 4), dtype=np.uint64))
        sels.append([(j % 4 == 0) and (j + 3 < ln) for j in range(ln)])
        total += ln
    bps = pyref.break_points_for(sels, max_rows)
    flat = np.concatenate([t for t in threads if len(t)])
    rc, want = orc.assign_witnesses(flat, np.array(bps, dtype=np.uint64), k, ncols)
    assert rc == 0
    got = h2b.assign_witnesses(ctx, threads, bps, k, ncols)
    assert np.array_equal(got, want)
    # too few columns: Rust panics (single_phase.rs:304) -> LayoutError
    with pytest.raises(h2b.LayoutError):
        h2b.assign_witnesses(ctx, threads, bps, k, len(bps))
    # no columns but cells present (single_phase.rs:279-286)
    with pytest.raises(h2b.LayoutError):
        h2b.assign_witnesses(ctx, threads, [], k, 0)
    # empty input
    got = h2b.assign_witnesses(ctx, [], [], k, 2)
    assert not got.any()
    # odd break points: walk semantics (break at row 0 of the first column; 0 never fires later)
    small = mont(list(range(1, 21)), R)
    for bp in ([0, 3], [3, 0, 2], [19], [25], [5, 5, 5]):
        rc, want = orc.assign_witnesses(small, np.array(bp, dtype=np.uint64), 5, 6)
        assert rc == 0
        assert np.array_equal(h2b.assign_witnesses(ctx, [small], bp, 5, 6), want), bp


def test_assign_lookups_and_rational(ctx, h2b):
    rng = np.random.default_rng(31)
    vals = mont(rand_ints(rng, 1000, R), R)
    for L in (1, 3, 4):
        rc, want = orc.assign_lookups(vals, 10, L)
        assert rc == 0
        assert np.array_equal(h2b.assign_lookups(ctx, vals, 10, L), want)
    with pytest.raises(h2b.LayoutError):
        h2b.assign_lookups(ctx, vals, 3, 2)
    num, den = mont(rand_ints(rng, 200, R), R), mont([0, 1] + rand_ints(rng, 198, R), R)
    assert np.array_equal(ctx.eval_rational(num, den), orc.eval_rational(num, den))


@pytest.mark.parametrize("n", [1, 5, 2048, 2049, 70001, 1 << 18])
def test_batch_invert_and_grand_product(ctx, h2b, n):
    """SURVEY.md §8(f) rank 2: the primitives of the permutation / lookup grand products"""
    rng = np.random.default_rng(900 + n % 97)
    A = rng.integers(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    A[:, 3] &= np.uint64((1 << 60) - 1)
    A[::7] = 0  # zeros are skipped by BatchInvert::batch_invert
    inv = ctx.batch_invert(A)
    assert np.array_equal(inv, orc.batch_invert(A))
    assert np.array_equal(orc.f_mul(orc.FR, inv[1:2], A[1:2]), mont([1], R)) if n > 1 else True
    F = rng.integers(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    F[:, 3] &= np.uint64((1 << 60) - 1)
    start = mont([3], R)[0]
    assert np.array_equal(ctx.grand_product(F, start), orc.grand_product(F, start))


def test_flex_gate_fold_and_vanishing(ctx, h2b):
    """SURVEY.md §8(f) rank 1, first slice.  (1) parity with the oracle on random data.  (2) end-to-end meaning: for a
    witness column that satisfies q*(a + b*c - out) on every row of the 2^k domain, the folded term evaluated on the
    extended coset is divisible by the vanishing polynomial X^n - 1; a broken witness is not."""
    rng = np.random.default_rng(62)
    k, j = 8, 5
    dom = h2b.EvaluationDomain(ctx, j, k)
    n, ek = 1 << k, dom.extended_k
    ne = 1 << ek

    def rnd(m):
        x = rng.integers(0, 1 << 62, size=(m, 4), dtype=np.int64).astype(np.uint64)
        x[:, 3] &= np.uint64((1 << 60) - 1)
        return x
    Q, A, ACC, y = rnd(ne), rnd(ne), rnd(ne), rnd(1)[0]
    assert np.array_equal(ctx.flex_gate_fold(Q, A, y, k, ek, ACC), orc.flex_gate_fold(Q, A, y, k, ek, ACC))
    # satisfied witness: gates at rows 0, 4, 8, ... (out = a + b*c), selector 1 there
    vals = rand_ints(rng, n, R)
    sel = [0] * n
    for r in range(0, n - 4, 4):
        vals[r + 3] = (vals[r] + vals[r + 1] * vals[r + 2]) % R
        sel[r] = 1
    q_ext = dom.coeff_to_extended(dom.lagrange_to_coeff(mont(sel, R)))
    zero = np.zeros((ne, 4), dtype=np.uint64)
    # 1 / t(X), t = X^n - 1, on the coset zeta*<w_ext>: t(zeta w^i) = zeta^n w^(n i) - 1 has period 2^(ek - k)
    we, zeta, per = pyref.omega_for(ek), pyref.ZETA, ne >> k
    tinv = [pow((pow(zeta, n, R) * pow(we, n * i, R) - 1) % R, -1, R) for i in range(per)]
    TI = mont([tinv[i % per] for i in range(ne)], R)

    def quotient_coeffs(values):
        a_ext = dom.coeff_to_extended(dom.lagrange_to_coeff(mont(values, R)))
        term = ctx.flex_gate_fold(q_ext, a_ext, y, k, ek, zero)
        full = h2b.EvaluationDomain(ctx, j, k)
        full.quotient_poly_degree = ne >> k  # keep all 2^ek coefficients
        return unmont(full.extended_to_coeff(orc.f_mul(orc.FR, term, TI)), R)
    hc = quotient_coeffs(vals)
    # deg(q * a * a) <= 3(n-1): exact division leaves deg(h) <= 2n - 3, everything above must be zero
    assert any(hc[: 2 * n]) and not any(hc[2 * n:])
    vals[3] = (vals[3] + 1) % R  # break one gate: no longer divisible, the high coefficients are non-zero
    assert any(quotient_coeffs(vals)[2 * n:])


def test_errors_do_not_cross_the_abi(ctx, h2b):
    with pytest.raises(h2b.H2BError):
        h2b.best_fft(ctx, np.zeros((1, 4), dtype=np.uint64), h2b.omega(0), 0) if False else ctx.check(
            h2b.lib.h2b_ntt_fr(ctx.h, None, 3, None, 0))
    with pytest.raises(h2b.H2BError):
        ctx.check(h2b.lib.h2b_msm_g1(ctx.h, None, 0, None, 4, None))


def test_assign_witnesses_from_assigned_records(ctx, h2b):
    """`Vec<Assigned<Fr>>` staging records (Zero / Trivial / Rational, halo2-base/src/lib.rs:157-188) in, columns out: the
    Rational cells go through the GPU's batched inversion (denominator 0 -> 0), then the literal walk's layout"""
    rng = np.random.default_rng(4100)
    k, ncols = 9, 3
    n = 1 << k
    N = 1200
    tags = rng.integers(0, 3, size=N)
    nums, dens = rand_ints(rng, N, R), rand_ints(rng, N, R)
    dens[5] = 0
    tags[5] = 2      # Rational with a zero denominator
    tags[6] = 0      # Zero whose payload fields hold garbage
    cells = np.zeros((N, 9), dtype=np.uint64)
    cells[:, 0] = tags
    cells[:, 1:5] = mont(nums, R)
    cells[:, 5:9] = mont(dens, R)
    want_vals = [0 if t == 0 else (v if t == 1 else (v * pow(d, -1, R) % R if d else 0)) for t, v, d in zip(tags, nums, dens)]
    bp = np.array([n - 21, n - 22], dtype=np.uint64)
    rc, want = orc.assign_witnesses(mont(want_vals, R), bp, k, ncols)
    assert rc == 0
    got = h2b.assign_witnesses_assigned(ctx, cells, bp, k, ncols)
    assert np.array_equal(got, want)
    # all-Trivial input takes the path without the inversion
    cells[:, 0] = 1
    rc, want = orc.assign_witnesses(mont(nums, R), bp, k, ncols)
    assert np.array_equal(h2b.assign_witnesses_assigned(ctx, cells, bp, k, ncols), want)
    # an unknown tag is rejected
    cells[7, 0] = 3
    with pytest.raises(h2b.H2BError):
        h2b.assign_witnesses_assigned(ctx, cells, bp, k, ncols)
    # many columns (> 64: the staged-span path) still match the walk
    k2, nc2 = 5, 70
    V = mont(rand_ints(rng, 31 + 39 * 30 + 25, R), R)  # 40 full columns (a break cell is copied into the next column) + 25 cells
    bp2 = np.array([30] * 40, dtype=np.uint64)
    rc, want = orc.assign_witnesses(V, bp2, k2, nc2)
    assert rc == 0
    assert np.array_equal(h2b.assign_witnesses(ctx, [V], bp2, k2, nc2), want)
