"""Python mirror of the reference-facing prover interface for the hot path (names and argument meaning follow
halo2-axiom 0.5.3 / halo2curves-axiom 0.7.3 as used by halo2-lib; SURVEY.md §8b):

    best_multiexp(coeffs, bases) -> G1                    halo2curves msm::best_multiexp
    ParamsKZG.commit / commit_lagrange                    poly::kzg::commitment::ParamsKZG
    best_fft(a, omega, log_n)                             arithmetic::best_fft
    EvaluationDomain(j, k).lagrange_to_coeff / coeff_to_extended / extended_to_coeff
    assign_witnesses(threads, break_points, ...)          halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312
    assign_lookups(values, ...)                           halo2-base/src/virtual_region/lookups.rs:130-155

Arrays are numpy uint64 in the `[u64;4]` little-endian Montgomery layout.  Everything computes on the GPU
through libh2b200.so; nothing here does field arithmetic on the CPU."""
from __future__ import annotations
import ctypes as C
import numpy as np
from ._capi import lib, H2B_OK, H2B_ERR_LAYOUT, H2B_ERR_UNSATISFIED, BASIS_MONOMIAL, BASIS_LAGRANGE


class H2BError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"h2b200 error {code}: {msg}")
        self.code = code


class LayoutError(H2BError):
    """Where the Rust code panics (out of columns / rows)."""


class ConstraintSystemFailure(H2BError):
    """plonk::Error::ConstraintSystemFailure (a lookup input that the table does not hold)."""


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    assert isinstance(a, np.ndarray) and a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"], "need contiguous uint64 ndarray"
    return C.c_void_p(a.ctypes.data)


def _u64(a, cols):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a.reshape(-1, cols)


class Context:
    """One per process / GPU (h2b_ctx)."""

    def __init__(self, device: int | list = 0):
        """device: one index, or a list of indices for a single-process device group (h2b_ctx_create_multi)"""
        h = C.c_void_p()
        if isinstance(device, (list, tuple)):
            ids = (C.c_int * len(device))(*device)
            rc = lib.h2b_ctx_create_multi(ids, len(device), C.byref(h))
            device = device[0]
        else:
            rc = lib.h2b_ctx_create(device, C.byref(h))
        if rc != H2B_OK:
            raise H2BError(rc, lib.h2b_last_error(None).decode())
        self.h = h
        self.device = device

    def check(self, rc: int):
        if rc != H2B_OK:
            msg = lib.h2b_last_error(self.h).decode()
            raise {H2B_ERR_LAYOUT: LayoutError, H2B_ERR_UNSATISFIED: ConstraintSystemFailure}.get(rc, H2BError)(rc, msg)

    def set_stream(self, cuda_stream: int | None):
        self.check(lib.h2b_ctx_set_stream(self.h, C.c_void_p(cuda_stream or 0)))

    def synchronize(self):
        self.check(lib.h2b_ctx_synchronize(self.h))

    def set_option(self, key: str, value: int):
        """tuning switches (h2b_ctx_set_option); results never depend on them"""
        self.check(lib.h2b_ctx_set_option(self.h, key.encode(), int(value)))

    @property
    def device_count(self) -> int:
        return int(lib.h2b_ctx_device_count(self.h))

    @property
    def kernel_launches(self) -> int:
        return int(lib.h2b_kernel_launches(self.h))

    def profile_enable(self, filt: str | None):
        self.check(lib.h2b_profile_enable(self.h, filt.encode() if filt else None))

    def profile_reset(self):
        self.check(lib.h2b_profile_reset(self.h))

    def profile_read(self, kernel: str) -> tuple[float, int]:
        ms, cnt = C.c_double(), C.c_uint64()
        self.check(lib.h2b_profile_read(self.h, kernel.encode(), C.byref(ms), C.byref(cnt)))
        return ms.value, int(cnt.value)

    def close(self):
        if self.h:
            lib.h2b_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- small group helpers
    def g1_sum(self, points_xyz) -> np.ndarray:
        p = _u64(points_xyz, 12)
        out = np.empty(12, dtype=np.uint64)
        self.check(lib.h2b_g1_sum(self.h, _ptr(p), len(p), _ptr(out)))
        return out

    def g1_normalize(self, points_xyz) -> np.ndarray:
        p = _u64(points_xyz, 12).copy()
        self.check(lib.h2b_g1_normalize(self.h, _ptr(p), len(p)))
        return p

    def g1_fixed_base_mul(self, base_xy, scalars) -> np.ndarray:
        b = _u64(base_xy, 8)
        s = _u64(scalars, 4)
        out = np.empty((len(s), 8), dtype=np.uint64)
        self.check(lib.h2b_g1_fixed_base_mul(self.h, _ptr(b), _ptr(s), len(s), _ptr(out)))
        return out

    def field_op(self, field: int, op: int, a, b=None) -> np.ndarray:
        a = _u64(a, 4)
        bb = _u64(b, 4) if b is not None else None
        out = np.empty_like(a)
        self.check(lib.h2b_test_field_op(self.h, field, op, _ptr(a), _ptr(bb), len(a), _ptr(out)))
        return out

    def batch_invert(self, a) -> np.ndarray:
        """ff `BatchInvert::batch_invert` (zeros stay zero); returns the inverted copy"""
        a = _u64(a, 4).copy()
        self.check(lib.h2b_batch_invert_fr(self.h, _ptr(a), len(a)))
        return a

    def grand_product(self, f, start) -> np.ndarray:
        """z[0] = start, z[i] = z[i-1] * f[i-1] (halo2 permutation / lookup product column)"""
        f = _u64(f, 4)
        st = _u64(start, 4)
        z = np.empty_like(f)
        self.check(lib.h2b_grand_product_fr(self.h, _ptr(f), _ptr(st), len(f), _ptr(z)))
        return z

    def flex_gate_fold(self, q_ext, a_ext, y, k: int, ext_k: int, acc) -> np.ndarray:
        """acc*y + q*(a + a(w X)*a(w^2 X) - a(w^3 X)) on the extended domain (halo2-base flex_gate/mod.rs:80-91)"""
        q, a, acc, yy = _u64(q_ext, 4), _u64(a_ext, 4), _u64(acc, 4).copy(), _u64(y, 4)
        self.check(lib.h2b_flex_gate_fold(self.h, _ptr(q), _ptr(a), _ptr(yy), k, ext_k, _ptr(acc)))
        return acc

    def eval_rational(self, num, den) -> np.ndarray:
        a, b = _u64(num, 4), _u64(den, 4)
        out = np.empty_like(a)
        self.check(lib.h2b_eval_rational(self.h, _ptr(a), _ptr(b), len(a), _ptr(out)))
        return out


def omega(k: int) -> np.ndarray:
    out = np.empty(4, dtype=np.uint64)
    rc = lib.h2b_domain_omega(k, _ptr(out))
    if rc != H2B_OK:
        raise H2BError(rc, "k out of range")
    return out


def best_multiexp(ctx: Context, coeffs, bases) -> np.ndarray:
    """halo2curves `best_multiexp(coeffs: &[Fr], bases: &[G1Affine]) -> G1`: ad-hoc bases, Jacobian result."""
    s, b = _u64(coeffs, 4), _u64(bases, 8)
    assert len(s) == len(b), "best_multiexp: coeffs.len() != bases.len()"  # Rust: assert_eq!
    out = np.empty(12, dtype=np.uint64)
    ctx.check(lib.h2b_msm_g1_bases(ctx.h, _ptr(b), _ptr(s), len(s), _ptr(out)))
    return out


def best_fft(ctx: Context, a, omega_m, log_n: int) -> np.ndarray:
    """halo2 `best_fft(a, omega, log_n)`; returns the transformed copy (Rust mutates in place)."""
    a = _u64(a, 4).copy()
    assert len(a) == 1 << log_n
    w = _u64(omega_m, 4)
    ctx.check(lib.h2b_ntt_fr(ctx.h, _ptr(a), log_n, _ptr(w), 0))
    return a


class ParamsKZG:
    """The base arrays of `ParamsKZG<Bn256>` (g, g_lagrange) resident on the GPU, sharded [begin, begin+count)."""

    def __init__(self, ctx: Context, k: int, g=None, g_lagrange=None, begin: int = 0, count: int | None = None,
                 device_ptrs: bool = False):
        self.ctx, self.k, self.n = ctx, k, 1 << k
        self.begin = begin
        self.count = (self.n - begin) if count is None else count
        h = C.c_void_p()
        if device_ptrs:
            rc = lib.h2b_srs_upload_dev(ctx.h, C.c_void_p(g or 0), C.c_void_p(g_lagrange or 0), k, begin, self.count, C.byref(h))
        else:
            gg = _u64(g, 8) if g is not None else None
            gl = _u64(g_lagrange, 8) if g_lagrange is not None else None
            for arr in (gg, gl):
                assert arr is None or len(arr) == self.n, "SRS arrays must hold all 2^k bases (the shard is cut inside)"
            rc = lib.h2b_srs_upload(ctx.h, _ptr(gg), _ptr(gl), k, begin, self.count, C.byref(h))
        ctx.check(rc)
        self.h = h
        cb, w = C.c_int(), C.c_int()
        lib.h2b_srs_info(self.h, C.byref(cb), C.byref(w))
        self.window_bits, self.windows = cb.value, w.value

    def _commit(self, basis: int, poly) -> np.ndarray:
        s = _u64(poly, 4)
        out = np.empty(12, dtype=np.uint64)
        self.ctx.check(lib.h2b_msm_g1(self.ctx.h, self.h, basis, _ptr(s), len(s), _ptr(out)))
        return out

    def commit(self, poly) -> np.ndarray:
        """ParamsKZG::commit(poly: coefficient form) -> G1 (monomial basis `g`)."""
        return self._commit(BASIS_MONOMIAL, poly)

    def commit_lagrange(self, poly) -> np.ndarray:
        """ParamsKZG::commit_lagrange(poly: Lagrange form) -> G1 (basis `g_lagrange`)."""
        return self._commit(BASIS_LAGRANGE, poly)

    def commit_batch(self, basis, polys) -> np.ndarray:
        """m commitments of one prover phase; `basis` is an int or a per-column list (0 monomial, 1 lagrange)."""
        cols = [_u64(p, 4) for p in polys]
        m = len(cols)
        out = np.empty((m, 12), dtype=np.uint64)
        ptrs = (C.c_void_p * m)(*[c.ctypes.data for c in cols])
        bs = (C.c_int * m)(*([basis] * m if isinstance(basis, int) else list(basis)))
        self.ctx.check(lib.h2b_msm_g1_batch(self.ctx.h, self.h, bs, ptrs, m, len(cols[0]) if m else 0, _ptr(out)))
        return out

    def commit_batch_dev(self, basis, d_scalar_ptrs, n: int, d_out: int):
        m = len(d_scalar_ptrs)
        ptrs = (C.c_void_p * m)(*d_scalar_ptrs)
        bs = (C.c_int * m)(*([basis] * m if isinstance(basis, int) else list(basis)))
        self.ctx.check(lib.h2b_msm_g1_batch_dev(self.ctx.h, self.h, bs, ptrs, m, n, C.c_void_p(d_out)))

    def commit_dev(self, basis: int, d_scalars: int, n: int, d_out: int):
        self.ctx.check(lib.h2b_msm_g1_dev(self.ctx.h, self.h, basis, C.c_void_p(d_scalars), n, C.c_void_p(d_out)))

    def close(self):
        if getattr(self, "h", None):
            lib.h2b_srs_destroy(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class EvaluationDomain:
    """halo2 `EvaluationDomain::new(j, k)`: j = cs.degree(); quotient_poly_degree = j - 1;
    extended_k = k + ceil(log2(j - 1)) (SURVEY.md Appendix B)."""

    def __init__(self, ctx: Context, j: int, k: int):
        self.ctx, self.k, self.n = ctx, k, 1 << k
        self.quotient_poly_degree = j - 1
        ek = k
        while (1 << ek) < self.n * self.quotient_poly_degree:
            ek += 1
        self.extended_k = ek

    def lagrange_to_coeff(self, a) -> np.ndarray:
        a = _u64(a, 4).copy()
        assert len(a) == self.n
        self.ctx.check(lib.h2b_lagrange_to_coeff(self.ctx.h, _ptr(a), self.k))
        return a

    def coeff_to_lagrange(self, a) -> np.ndarray:
        a = _u64(a, 4).copy()
        assert len(a) == self.n
        self.ctx.check(lib.h2b_coeff_to_lagrange(self.ctx.h, _ptr(a), self.k))
        return a

    def lagrange_to_coeff_many(self, cols) -> list:
        """`cols.iter().map(|c| domain.lagrange_to_coeff(c))`, pipelined over PCIe"""
        arrs = [_u64(a, 4).copy() for a in cols]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        self.ctx.check(lib.h2b_lagrange_to_coeff_batch(self.ctx.h, ptrs, len(arrs), self.k))
        return arrs

    def lagrange_to_coeff_and_extended_many(self, cols) -> tuple:
        """(coefficients, coset evaluations) of every column: one fused, PCIe-pipelined call"""
        arrs = [_u64(a, 4).copy() for a in cols]
        outs = [np.empty((1 << self.extended_k, 4), dtype=np.uint64) for _ in arrs]
        pin = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pout = (C.c_void_p * len(arrs))(*[o.ctypes.data for o in outs])
        self.ctx.check(lib.h2b_lagrange_to_coeff_and_extended_batch(self.ctx.h, pin, len(arrs), self.k, self.extended_k, pout))
        return arrs, outs

    def coeff_to_extended_many(self, cols) -> list:
        arrs = [_u64(a, 4) for a in cols]
        outs = [np.empty((1 << self.extended_k, 4), dtype=np.uint64) for _ in arrs]
        pin = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pout = (C.c_void_p * len(arrs))(*[o.ctypes.data for o in outs])
        self.ctx.check(lib.h2b_coeff_to_extended_batch(self.ctx.h, pin, len(arrs), self.n, self.extended_k, pout))
        return outs

    def coeff_to_extended(self, a) -> np.ndarray:
        a = _u64(a, 4)
        assert len(a) == self.n
        out = np.empty((1 << self.extended_k, 4), dtype=np.uint64)
        self.ctx.check(lib.h2b_coeff_to_extended(self.ctx.h, _ptr(a), len(a), self.extended_k, _ptr(out)))
        return out

    def extended_to_coeff(self, a) -> np.ndarray:
        a = _u64(a, 4).copy()
        assert len(a) == 1 << self.extended_k
        self.ctx.check(lib.h2b_extended_to_coeff(self.ctx.h, _ptr(a), self.extended_k))
        return a[: self.n * self.quotient_poly_degree]  # `a.values.truncate(n * quotient_poly_degree)`


def assign_witnesses(ctx: Context, threads, break_points, k: int, ncols: int) -> np.ndarray:
    """`assign_witnesses(threads, basic_gates, region, break_points)`: threads = list of (len_i x 4) limb arrays
    (ctx.advice of each Context, Trivial payloads); returns ncols x 2^k x 4.  Raises LayoutError where Rust panics."""
    parts = [_u64(t, 4) for t in threads if len(t)]
    vcol = np.concatenate(parts) if parts else np.zeros((0, 4), dtype=np.uint64)
    bp = np.ascontiguousarray(break_points, dtype=np.uint64).reshape(-1)
    cols = np.empty((ncols, 1 << k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_assign_columns(ctx.h, _ptr(vcol) if len(vcol) else None, len(vcol), _ptr(bp) if len(bp) else None,
                                     len(bp), k, ncols, _ptr(cols) if ncols else None))
    return cols


def assign_witnesses_assigned(ctx: Context, cells, break_points, k: int, ncols: int) -> np.ndarray:
    """`assign_witnesses` fed with `Assigned<Fr>` staging records: cells = N x 9 uint64 (tag, numerator[4], denominator[4]),
    tag 0 Zero / 1 Trivial / 2 Rational (halo2-base/src/lib.rs:157-188); the Rational cells are batch-inverted on the GPU"""
    c = np.ascontiguousarray(cells, dtype=np.uint64).reshape(-1, 9)
    bp = np.ascontiguousarray(break_points, dtype=np.uint64).reshape(-1)
    cols = np.empty((ncols, 1 << k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_assign_columns_assigned(ctx.h, _ptr(c) if len(c) else None, len(c), _ptr(bp) if len(bp) else None, len(bp), k, ncols,
                                              _ptr(cols) if ncols else None))
    return cols


def apply_rational_dev(ctx: Context, d_values: int, N: int, d_index: int, d_den: int, R: int, d_status: int):
    """halo2-base form, device pointers, asynchronous: values[index[i]] *= den[i]^-1 (d = 0 -> 0), den inverted in place;
    the verdict word at d_status (u32) gets bit 0 for an index >= N, bit 1 for indices that do not strictly increase"""
    vp = C.c_void_p
    ctx.check(lib.h2b_apply_rational_dev(ctx.h, vp(d_values), N, vp(d_index), vp(d_den), R, vp(d_status)))


def assign_lookups_indexed_dev(ctx: Context, d_values: int, N: int, d_index: int, n_lookup: int, k: int, L: int, d_cols: int,
                               d_status: int):
    """`assign_raw` from virtual-column indices, device pointers, asynchronous: lookup cell j = values[index[j]] goes to
    column j mod L, row j div L of d_cols (L x 2^k cells); bit 0 of the verdict word at d_status for an index >= N"""
    vp = C.c_void_p
    ctx.check(lib.h2b_assign_lookups_indexed_dev(ctx.h, vp(d_values), N, vp(d_index), n_lookup, k, L, vp(d_cols), vp(d_status)))


def assign_lookups(ctx: Context, values, k: int, L: int) -> np.ndarray:
    v = _u64(values, 4)
    cols = np.empty((L, 1 << k, 4), dtype=np.uint64)
    ctx.check(lib.h2b_assign_lookups(ctx.h, _ptr(v) if len(v) else None, len(v), k, L, _ptr(cols) if L else None))
    return cols
