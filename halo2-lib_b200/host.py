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
import os
import numpy as np
from ._capi import lib, H2B_OK, H2B_ERR_ARG, H2B_ERR_LAYOUT, H2B_ERR_UNSATISFIED, BASIS_MONOMIAL, BASIS_LAGRANGE


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
        """element-wise test hook h2b_test_field_op; op 10 takes 2n rows in `a` and `b` ((a_i, b_i) then (a_{n+i}, b_{n+i}))
        and returns n rows"""
        a = _u64(a, 4)
        bb = _u64(b, 4) if b is not None else None
        n = len(a)
        if op == 10:
            assert n % 2 == 0 and (bb is None or len(bb) == n), "field_op 10: a and b hold 2n rows each"
            n //= 2
        out = np.empty((n, 4), dtype=np.uint64)
        self.check(lib.h2b_test_field_op(self.h, field, op, _ptr(a), _ptr(bb), n, _ptr(out)))
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


_P_MOD = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
# the G1 generator (1, 2), Montgomery limbs: the base of ParamsKZG::setup
G1_GENERATOR = np.array([(v << 256) % _P_MOD >> (64 * i) & 0xFFFFFFFFFFFFFFFF for v in (1, 2) for i in range(4)], dtype=np.uint64)


class _DeviceBuffer:
    """`elems` x 32 bytes of device memory (one h2b_poly); an affine G1 point takes two elements"""

    def __init__(self, ctx: Context, elems: int):
        self.ctx, h = ctx, C.c_void_p()
        ctx.check(lib.h2b_poly_alloc(ctx.h, elems, C.byref(h)))
        self.h, self.ptr = h, int(lib.h2b_poly_device_ptr(h))

    def free(self):
        if self.h:
            lib.h2b_poly_free(self.ctx.h, self.h)
            self.h = None


def seeded_tau(seed: bytes = bytes(32)) -> np.ndarray:
    """tau of `ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed))` (gen_srs: 32 zero bytes), Montgomery limbs"""
    s = np.frombuffer(bytes(seed), dtype=np.uint8).copy()
    assert len(s) == 32, "the seed is 32 bytes"
    t = np.zeros(4, dtype=np.uint64)
    rc = lib.h2b_srs_seeded_tau(_ptr8(s), _ptr(t))
    if rc != H2B_OK:
        raise H2BError(rc, "h2b_srs_seeded_tau")
    return t


def g2_generator_mul(tau) -> tuple[bytes, bytes]:
    """(g2 | s_g2 compressed, g2 | s_g2 raw) with s_g2 = tau * g2: the G2 pair of a params image in both formats"""
    t = _u64(tau, 4).reshape(4)
    proc, raw = np.zeros(128, dtype=np.uint8), np.zeros(256, dtype=np.uint8)
    rc = lib.h2b_g2_generator_mul(_ptr(t), _ptr8(proc), _ptr8(raw))
    if rc != H2B_OK:
        raise H2BError(rc, "h2b_g2_generator_mul: tau must be below r")
    return proc.tobytes(), raw.tobytes()


def _ptr8(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def _image_view(view, image: np.ndarray) -> tuple:
    k, off = C.c_uint32(), [C.c_size_t() for _ in range(4)]
    if view(_ptr8(image), len(image), C.byref(k), *[C.byref(o) for o in off]) != H2B_OK:
        raise H2BError(H2B_ERR_ARG, "not a params image")
    return k.value, [o.value for o in off]


class ParamsKZG:
    """The base arrays of `ParamsKZG<Bn256>` (g, g_lagrange) resident on the GPU, sharded [begin, begin+count).

    Params made by setup_seeded / gen_srs / read_downsized also keep g and g_lagrange themselves on the device (whole, not
    sharded) and the G2 pair (g2, s_g2), so that they can be written (`ParamsKZG::write`) and downsized."""

    def __init__(self, ctx: Context, k: int, g=None, g_lagrange=None, begin: int = 0, count: int | None = None,
                 device_ptrs: bool = False):
        self.ctx, self.k, self.n = ctx, k, 1 << k
        self.begin = begin
        self.count = (self.n - begin) if count is None else count
        self._g = self._gl = None  # _DeviceBuffer of setup_seeded / read_downsized
        self.g2_processed = self.g2_raw = None  # g2 | s_g2 in the Processed (128 bytes) and RawBytes (256 bytes) encodings
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

    # ---- creating, writing and downsizing halo2-lib's params (gen_srs, ParamsKZG::write, Params::downsize)
    @classmethod
    def _resident(cls, ctx: Context, k: int, g: _DeviceBuffer, gl: _DeviceBuffer, g2_processed, g2_raw):
        try:
            params = cls(ctx, k, g.ptr, gl.ptr, device_ptrs=True)
        except Exception:
            g.free(); gl.free()
            raise
        params._g, params._gl, params.g2_processed, params.g2_raw = g, gl, g2_processed, g2_raw
        return params

    @classmethod
    def setup_seeded(cls, ctx: Context, k: int, seed: bytes = bytes(32)) -> "ParamsKZG":
        """`ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed))`, what gen_srs creates: g, g_lagrange at halo2-lib's tau on the
        device, the G2 pair on the host"""
        tau = seeded_tau(seed)
        g, gl = _DeviceBuffer(ctx, 2 << k), _DeviceBuffer(ctx, 2 << k)
        try:
            ctx.check(lib.h2b_srs_setup_dev(ctx.h, _ptr(tau), _ptr(G1_GENERATOR), k, C.c_void_p(g.ptr), C.c_void_p(gl.ptr)))
        except Exception:
            g.free(); gl.free()
            raise
        return cls._resident(ctx, k, g, gl, *g2_generator_mul(tau))

    @classmethod
    def read_downsized(cls, ctx: Context, image, k: int | None = None) -> "ParamsKZG":
        """`read_params(K).downsize(k)` from a SerdeFormat::Processed image: only the first 2^k encodings of g are decompressed,
        g_lagrange is rebuilt from them (g_to_lagrange) and G2 is kept; the 2^K bases never reach the device.  H2BError
        (H2B_ERR_ARG) for a malformed image or an invalid encoding."""
        img = np.frombuffer(bytes(image), dtype=np.uint8) if not isinstance(image, np.ndarray) else np.ascontiguousarray(image, dtype=np.uint8)
        big_k, (og, _, og2, _) = _image_view(lib.h2b_params_processed_view, img)
        k = big_k if k is None else k
        if k > big_k:
            raise H2BError(H2B_ERR_ARG, f"downsize: k = {k} above the image's k = {big_k}")
        n = 1 << k
        enc, g, gl = _DeviceBuffer(ctx, n), _DeviceBuffer(ctx, 2 * n), _DeviceBuffer(ctx, 2 * n)
        try:
            ctx.check(lib.h2b_poly_upload(ctx.h, enc.h, 0, _ptr8(img[og:og + 32 * n]), n))
            bad = C.c_size_t()
            ctx.check(lib.h2b_g1_decompress_dev(ctx.h, C.c_void_p(enc.ptr), n, C.c_void_p(g.ptr), C.byref(bad)))
            if bad.value:
                raise H2BError(H2B_ERR_ARG, "read_params: the params image holds an invalid G1 encoding")
            ctx.check(lib.h2b_g_to_lagrange_dev(ctx.h, C.c_void_p(g.ptr), k, C.c_void_p(gl.ptr)))
        except Exception:
            g.free(); gl.free()
            raise
        finally:
            enc.free()
        return cls._resident(ctx, k, g, gl, img[og2:og2 + 128].tobytes(), None)

    @classmethod
    def read(cls, ctx: Context, image) -> "ParamsKZG":
        """`ParamsKZG::read` of a SerdeFormat::Processed image: the SRS handle through h2b_srs_read_processed (the bases are
        not kept, so these params cannot be written or downsized); H2BError (H2B_ERR_ARG) for a malformed image or an invalid
        encoding"""
        img = np.frombuffer(bytes(image), dtype=np.uint8) if not isinstance(image, np.ndarray) else np.ascontiguousarray(image, dtype=np.uint8)
        h = C.c_void_p()
        ctx.check(lib.h2b_srs_read_processed(ctx.h, _ptr8(img), len(img), 0, 0, C.byref(h)))
        params = cls.__new__(cls)
        k, (_, _, og2, _) = _image_view(lib.h2b_params_processed_view, img)
        params.ctx, params.k, params.n, params.begin, params.count, params.h = ctx, k, 1 << k, 0, 1 << k, h
        params._g = params._gl = params.g2_raw = None
        params.g2_processed = img[og2:og2 + 128].tobytes()
        cb, w = C.c_int(), C.c_int()
        lib.h2b_srs_info(h, C.byref(cb), C.byref(w))
        params.window_bits, params.windows = cb.value, w.value
        return params

    def _need_bases(self, what: str):
        if self._g is None:
            raise H2BError(H2B_ERR_ARG, f"{what}: these params do not keep their bases on the device (use setup_seeded / read_downsized)")

    def write(self, format: str = "processed") -> bytes:
        """`ParamsKZG::write` in SerdeFormat::Processed ("processed") or RawBytes ("raw"): u32 LE k | g | g_lagrange | g2 | s_g2"""
        self._need_bases("write")
        fn, g2 = {"processed": (lib.h2b_params_write_processed, self.g2_processed), "raw": (lib.h2b_params_write_raw, self.g2_raw)}[format]
        if g2 is None:
            raise H2BError(H2B_ERR_ARG, f"write: the {format} encoding of G2 is not known for params read from an image")
        ln = C.c_size_t()
        self.ctx.check(fn(self.ctx.h, None, None, self.k, None, None, C.byref(ln)))
        out = np.empty(ln.value, dtype=np.uint8)
        g2a = np.frombuffer(g2, dtype=np.uint8).copy()
        self.ctx.check(fn(self.ctx.h, C.c_void_p(self._g.ptr), C.c_void_p(self._gl.ptr), self.k, _ptr8(g2a), _ptr8(out), C.byref(ln)))
        return out.tobytes()

    def downsize(self, k: int):
        """`Params::downsize(k)` in place: g keeps its first 2^k points, g_lagrange is rebuilt from them, G2 stays"""
        self._need_bases("downsize")
        if k > self.k:
            raise H2BError(H2B_ERR_ARG, f"downsize: k = {k} above the params' k = {self.k}")
        n = 1 << k
        g, gl = _DeviceBuffer(self.ctx, 2 * n), _DeviceBuffer(self.ctx, 2 * n)
        try:
            self.ctx.check(lib.h2b_poly_copy_dev(self.ctx.h, C.c_void_p(g.ptr), C.c_void_p(self._g.ptr), 2 * n))
            self.ctx.check(lib.h2b_g_to_lagrange_dev(self.ctx.h, C.c_void_p(g.ptr), k, C.c_void_p(gl.ptr)))
            h = C.c_void_p()
            self.ctx.check(lib.h2b_srs_upload_dev(self.ctx.h, C.c_void_p(g.ptr), C.c_void_p(gl.ptr), k, 0, n, C.byref(h)))
        except Exception:
            g.free(); gl.free()
            raise
        lib.h2b_srs_destroy(self.ctx.h, self.h)
        self._g.free(); self._gl.free()
        self.h, self._g, self._gl, self.k, self.n, self.count = h, g, gl, k, n, n
        cb, w = C.c_int(), C.c_int()
        lib.h2b_srs_info(self.h, C.byref(cb), C.byref(w))
        self.window_bits, self.windows = cb.value, w.value

    def close(self):
        if getattr(self, "h", None):
            lib.h2b_srs_destroy(self.ctx.h, self.h)
            self.h = None
        for b in (getattr(self, "_g", None), getattr(self, "_gl", None)):
            if b is not None:
                b.free()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def srs_path(k: int, dir: str | None = None) -> str:
    """where gen_srs caches the params of 2^k rows: $PARAMS_DIR (or ./params) / kzg_bn254_{k}.srs"""
    return os.path.join(dir if dir is not None else os.environ.get("PARAMS_DIR", "./params"), f"kzg_bn254_{k}.srs")


def gen_srs(ctx: Context, k: int, dir: str | None = None) -> ParamsKZG:
    """halo2-base `gen_srs(k)` = read_or_create_srs: read the cached SerdeFormat::Processed params when the file exists
    (ParamsKZG.read), else create them with setup_seeded (zero seed), create the directory and write the file"""
    path = srs_path(k, dir)
    if os.path.exists(path):
        with open(path, "rb") as f:
            return ParamsKZG.read(ctx, f.read())
    params = ParamsKZG.setup_seeded(ctx, k)
    try:
        image = params.write("processed")
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        with open(path, "wb") as f:
            f.write(image)
    except Exception:
        params.close()
        raise
    return params


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
