"""The field arithmetic of the kernels (csrc/field.cuh) on raw limb patterns, bit for bit against plain Python integers
(tests/field_edges.py), and the group-law kernels on points whose raw coordinates are such patterns.

Every op of h2b_test_field_op runs on every ordered pair of the fixed family, on 2^18 limb-pattern samples, on operands
close to m and on products aimed at both sides of the final conditional subtraction.  A failure names the op, the field,
the sample group and the first failing operands in hex."""
import numpy as np
import pytest
import field_edges as fe
from oracle import pyref
from util import affine_to_limbs, jac_limbs_to_affine

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


@pytest.mark.parametrize("op", sorted(fe.OPS), ids=[f"{k}-{fe.OPS[k]}" for k in sorted(fe.OPS)])
@pytest.mark.parametrize("field", ["Fq", "Fr"])
def test_field_op_on_raw_limb_edges(ctx, field, op):
    which, m = fe.FIELDS[field]
    errors = []
    for group, tuples in fe.samples(field)[op].items():
        a, b = fe.pack(op, tuples)
        got = fe.from_limbs(ctx.field_op(which, op, a, b))
        msg = fe.first_mismatch(op, field, group, tuples, got, fe.reference_many(op, m, tuples))
        if msg:
            errors.append(msg)
    assert not errors, "\n".join(errors)


# ------------------------------------------------------------------------------------------------ group law
def _edge_points(n):
    """affine points whose Montgomery x limbs come from the fixed and limb-pattern families of Fq"""
    raw = fe.fixed_family(P) + fe.pattern_family(P, 4 * n, 0xC0FFEE)
    return fe.curve_points(raw, n)


def _jacobian(pts, zs):
    """(x z^2, y z^3, z) Montgomery limbs with the given raw z limbs (z = 0 only for the identity)"""
    out = np.zeros((len(pts), 12), dtype=np.uint64)
    rinv = pow(fe.W, -1, P)
    for i, (pt, zr) in enumerate(zip(pts, zs)):
        if pt is None:
            out[i, 4:8] = fe.to_limbs([fe.W % P])[0]
            continue
        z = zr * rinv % P
        x, y = pt[0] * z * z % P, pt[1] * z * z * z % P
        out[i] = fe.to_limbs([x * fe.W % P, y * fe.W % P, zr]).reshape(12)
    return out


def _sum(pts):
    acc = None
    for p in pts:
        acc = pyref.g1_add(acc, p)
    return acc


def test_g1_sum_on_edge_coordinates(ctx):
    """the quad formulas of g1_sum on points with extreme raw x and extreme raw z, including P + P and P + (-P)"""
    pts = _edge_points(48)
    zs = [z for z in fe.fixed_family(P) if z] + fe.pattern_family(P, 64, 0xBEEF)
    zs = [zs[i % len(zs)] for i in range(len(pts))]
    assert all(pyref.is_on_curve(p) for p in pts)
    for sel in (pts, pts[:2], pts[:1] * 2, [pts[0], pyref.g1_neg(pts[0])], pts[:3] + [None] + pts[3:9]):
        got = jac_limbs_to_affine(ctx.g1_sum(_jacobian(sel, zs)))
        assert got == _sum(sel), [hex(p[0] * fe.W % P) for p in sel if p]
    for i in range(0, len(pts) - 1, 2):  # pairs: every point once as the first and once as the second operand
        pair = [pts[i], pts[i + 1]]
        assert jac_limbs_to_affine(ctx.g1_sum(_jacobian(pair, zs[i:i + 2]))) == _sum(pair), hex(pts[i][0] * fe.W % P)


def test_fixed_base_mul_with_edge_bases(ctx):
    pts = _edge_points(8)
    scalars = [1, 2, 3, R - 1, R - 2, (R - 1) // 2, 0xFFFFFFFF, 1 << 128]
    sm = fe.to_limbs([s * fe.W % R for s in scalars])
    for pt in pts:
        got = ctx.g1_fixed_base_mul(affine_to_limbs([pt])[0], sm)
        want = affine_to_limbs([pyref.g1_mul(s, pt) for s in scalars])
        assert np.array_equal(got, want), hex(pt[0] * fe.W % P)


def test_msm_and_commit_with_edge_bases(ctx, h2b):
    """best_multiexp and ParamsKZG.commit (its table: k_precompute_level's doubling chain and inversions) over 2^6 bases
    with extreme raw coordinates"""
    k = 6
    n = 1 << k
    pts = _edge_points(n)
    assert len(pts) == n
    rng = np.random.default_rng(61)
    sc = [int.from_bytes(rng.bytes(32), "little") % R for _ in range(n)]
    sc[:4] = [1, R - 1, 0, 2]
    S = fe.to_limbs([s * fe.W % R for s in sc])
    B = affine_to_limbs(pts)
    want = pyref.msm_naive(sc, pts)
    assert jac_limbs_to_affine(h2b.best_multiexp(ctx, S, B)) == want
    params = h2b.ParamsKZG(ctx, k, g=B)
    try:
        assert jac_limbs_to_affine(params.commit(S)) == want
    finally:
        params.close()


def test_compress_decompress_edge_points(ctx):
    import ctypes as C
    from halo2_lib_b200._capi import lib
    pts = _edge_points(64) + [None]
    B = affine_to_limbs(pts)
    enc = np.zeros((len(pts), 32), dtype=np.uint8)
    ctx.check(lib.h2b_g1_compress(ctx.h, C.c_void_p(B.ctypes.data), len(pts), C.c_void_p(enc.ctypes.data)))
    assert [bytes(e) for e in enc] == [pyref.g1_compress(p) for p in pts]
    back, bad = np.zeros_like(B), C.c_size_t(7)
    ctx.check(lib.h2b_g1_decompress(ctx.h, C.c_void_p(enc.ctypes.data), len(pts), C.c_void_p(back.ctypes.data), C.byref(bad)))
    assert bad.value == 0 and np.array_equal(back, B)
