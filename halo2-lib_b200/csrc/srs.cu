// srs.cu — keygen-side SRS utilities for sm_90a (SURVEY.md §8(f) rank 3):
//   g_to_lagrange   halo2-axiom 0.5.3 `poly/kzg/commitment.rs::g_to_lagrange` = best_fft over G1 with omega^-1, every
//                   point scaled by 2^-k, batch-normalised:  g_lagrange[i] = (1/n) sum_j omega^(-i j) g[j]
//   srs_setup       `ParamsKZG::setup` for a caller-supplied tau: g[i] = tau^i G, g_lagrange[i] = L_i(tau) G with
//                   L_i(tau) = (tau^n - 1)/n * omega^i / (tau - omega^i)
//   on-curve check  y^2 = x^3 + 3 or (0,0) for points read from a params file (`ParamsKZG::read`,
//                   halo2-base/src/utils/mod.rs:401-424)
// (not vendored; restated from the definitions — the outputs are unique group elements).
//
// The group FFT is radix-2 decimation in time on XYZZ points in HBM: n/2 butterflies per stage, each one scalar
// multiplication by a twiddle plus two point additions — integer-multiplier bound, run once per SRS.  The scalar
// multiplication uses the curve's endomorphism (GLV): phi(x, y) = (beta x, y) = lambda (x, y), so
// tw * P = k1 * P + k2 * phi(P) with |k1|, |k2| < 2^127 (k_glv_decompose, once per distinct twiddle), evaluated jointly
// with 2-bit windows over a 16-entry table i*P + j*phi(P): 128 doublings + <= 64 additions + 13 table additions
// (~2.2k Montgomery products) instead of 254 + ~127 (~4.1k) for the plain double-and-add.
#include "h2b_internal.cuh"
#include "curve.cuh"
#include "fr_domain_consts.inc"

namespace h2b {

// ---------------------------------------------------------------- compressed points (SerdeFormat::Processed)
// halo2curves `G1Affine::from_bytes` as `ParamsKZG::read` applies it to a `kzg_bn254_{k}.srs` file written in
// SerdeFormat::Processed (reference call sites halo2-base/src/utils/mod.rs:401-435): 32 bytes = x, little-endian,
// canonical; the two spare bits of the last byte carry bit 7 = point at infinity, bit 6 = parity of y (LSB of the
// canonical y).  [halo2curves-axiom 0.7.3 is not vendored: the flag positions are recalled, see DESIGN.md §2.]
// y = sqrt(x^3 + 3) = (x^3 + 3)^((p + 1) / 4) since p = 3 mod 4; a non-residue, an x >= p, or an infinity flag on a
// non-zero x is an invalid encoding.  out = (x, y) Montgomery, (0, 0) for the identity; invalid -> (0, 0) and counted.
__device__ __forceinline__ Fq fq_sqrt_candidate(const Fq& a) {
    // (p + 1) / 4, little-endian 32-bit limbs
    const u32 e[8] = {0xb61f3f52u, 0x4f082305u, 0x5a1c72a3u, 0x65e05aa4u, 0xa0605617u, 0x6e14116du, 0xb84c680au, 0x0c19139cu};
    Fq acc = Fq::one();
#pragma unroll 1
    for (int limb = 7; limb >= 0; limb--) {
        u32 v = 0;
#pragma unroll
        for (int t = 0; t < 8; t++)
            if (t == limb) v = e[t];
#pragma unroll 1
        for (int bit = 31; bit >= 0; bit--) {
            acc = acc.sqr();
            if ((v >> bit) & 1) acc = acc * a;
        }
    }
    return acc;
}
__global__ void __launch_bounds__(128) k_g1_decompress(const uint8_t* __restrict__ bytes, size_t n, Affine* __restrict__ out,
                                                       unsigned long long* __restrict__ invalid) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* q = reinterpret_cast<const uint4*>(bytes + 32 * i);
    const uint4 lo = __ldg(q), hi = __ldg(q + 1);
    Fq x;
    x.l[0] = lo.x; x.l[1] = lo.y; x.l[2] = lo.z; x.l[3] = lo.w;
    x.l[4] = hi.x; x.l[5] = hi.y; x.l[6] = hi.z; x.l[7] = hi.w;
    const bool inf = x.l[7] & (H2B_G1_FLAG_IDENTITY << 24), odd = x.l[7] & (H2B_G1_FLAG_Y_ODD << 24);
    x.l[7] &= ~((H2B_G1_FLAG_IDENTITY | H2B_G1_FLAG_Y_ODD) << 24);
    Affine r;
    r.x = Fq::zero();
    r.y = Fq::zero();
    bool bad = false;
    if (inf) {
        bad = !x.is_zero() || odd;
    } else {
        // canonical: x < p
        bool lt = false;
        for (int t = 7; t >= 0; t--) {
            if (x.l[t] != FqParams::MOD(t)) { lt = x.l[t] < FqParams::MOD(t); break; }
        }
        if (!lt) bad = true;
        else {
            const Fq xm = x.to_mont();
            Fq three = Fq::one();
            three = three + three + Fq::one();
            const Fq rhs = xm.sqr() * xm + three;
            Fq y = fq_sqrt_candidate(rhs);
            if (!(y.sqr() == rhs)) bad = true;
            else {
                if ((y.from_mont().l[0] & 1u) != (odd ? 1u : 0u)) y = y.neg();
                r.x = xm;
                r.y = y;
            }
        }
    }
    if (bad) atomicAdd(invalid, 1ull);
    r.store(out + i);
}
// the inverse of k_g1_decompress (`G1Affine::to_bytes`, what `ParamsKZG::write` emits in SerdeFormat::Processed): canonical x
// little-endian, bit 6 of byte 31 = parity of the canonical y; the identity (0, 0) -> all zero but bit 7 of byte 31.  Two
// from_mont per point and nothing else: 64 bytes read, 32 written, bound by HBM.
__global__ void __launch_bounds__(256) k_g1_compress(const Affine* __restrict__ pts, size_t n, uint8_t* __restrict__ bytes) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Affine p = Affine::load(pts + i);
    uint4 lo = make_uint4(0, 0, 0, 0), hi = make_uint4(0, 0, 0, H2B_G1_FLAG_IDENTITY << 24);
    if (!p.is_identity()) {
        const Fq x = p.x.from_mont(), y = p.y.from_mont();
        lo = make_uint4(x.l[0], x.l[1], x.l[2], x.l[3]);
        hi = make_uint4(x.l[4], x.l[5], x.l[6], x.l[7] | ((y.l[0] & 1u) ? H2B_G1_FLAG_Y_ODD << 24 : 0u));
    }
    uint4* q = reinterpret_cast<uint4*>(bytes + 32 * i);
    q[0] = lo;
    q[1] = hi;
}

// ---------------------------------------------------------------- GLV scalar multiplication
// lambda = 0xb3c4d79d41a917585bfc41088d8daaa78b17ea66b99c90dd (lambda^2 + lambda + 1 = 0 mod r) acts on G1 as
// phi(x, y) = (beta x, y), beta = 0x59e26bcea0d48bacd4f263f1acdb5c4f5763473177fffffe (checked against the oracle's
// scalar multiplication in tests/test_oracle_srs.py).  Lattice basis of {(a, b): a + b lambda = 0 mod r} from the
// extended Euclid on (r, lambda):  v1 = (a1, -|b1|), v2 = (a2, b2), det = r.  For a scalar k:
//     c1 = floor(k g1 / 2^256), c2 = floor(k g2 / 2^256),  g1 = floor(2^256 b2 / r), g2 = floor(2^256 |b1| / r),
//     k1 = k - c1 a1 - c2 a2,   k2 = c1 |b1| - c2 b2,      k = k1 + k2 lambda (mod r),  |k1|, |k2| < 2^127.
struct GlvScalar {
    u32 k1[4], k2[4];  // magnitudes
    u32 neg;           // bit 0: k1 < 0, bit 1: k2 < 0
    u32 pad[3];
};
template <int NA, int NB>
__device__ __forceinline__ void mp_mul(const u32* a, const u32* b, u32* out) {  // out[NA + NB] = a * b
#pragma unroll
    for (int i = 0; i < NA + NB; i++) out[i] = 0;
#pragma unroll
    for (int i = 0; i < NA; i++) {
        u64 carry = 0;
#pragma unroll
        for (int j = 0; j < NB; j++) {
            const u64 t = (u64)a[i] * b[j] + out[i + j] + carry;
            out[i + j] = (u32)t;
            carry = t >> 32;
        }
        out[i + NB] = (u32)carry;
    }
}
template <int N>
__device__ __forceinline__ void mp_sub(u32* a, const u32* b) {  // a -= b (mod 2^(32 N))
    u64 borrow = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
        const u64 t = (u64)a[i] - b[i] - borrow;
        a[i] = (u32)t;
        borrow = (t >> 32) & 1;
    }
}
template <int N>
__device__ __forceinline__ bool mp_abs(u32* a) {  // two's complement -> magnitude; returns the sign
    const bool neg = a[N - 1] >> 31;
    if (neg) {
        u64 carry = 1;
#pragma unroll
        for (int i = 0; i < N; i++) {
            const u64 t = (u64)(~a[i]) + carry;
            a[i] = (u32)t;
            carry = t >> 32;
        }
    }
    return neg;
}
__device__ __forceinline__ GlvScalar glv_decompose(const Fr& k) {  // k canonical
    const u32 A1[2] = {0x94d213e3u, 0x89d32568u};
    const u32 B1[4] = {0x7d4f1128u, 0x8211bbebu, 0xeeb859fcu, 0x6f4d8248u};  // |b1|, b1 < 0
    const u32 A2[4] = {0x1221250bu, 0x0be4e154u, 0xeeb859fdu, 0x6f4d8248u};
    const u32 B2[2] = {0x94d213e3u, 0x89d32568u};
    const u32 G1[3] = {0xc7e0b3d7u, 0xd91d232eu, 0x00000002u};
    const u32 G2[5] = {0x391eb18du, 0x7a7bd9d4u, 0xa773d2cfu, 0x4ccef014u, 0x00000002u};
    u32 t1[11], t2[13];
    mp_mul<8, 3>(k.l, G1, t1);
    mp_mul<8, 5>(k.l, G2, t2);
    const u32* c1 = t1 + 8;  // < 2^64 (k < 2^254, g1 < 2^66); 3 limbs kept, the top one is 0
    const u32* c2 = t2 + 8;  // < 2^128; 5 limbs kept, the top one is 0
    // k1 = k - c1 a1 - c2 a2 over 9 limbs (two's complement)
    u32 k1[9], p1[5], p2[9];
#pragma unroll
    for (int i = 0; i < 8; i++) k1[i] = k.l[i];
    k1[8] = 0;
    mp_mul<3, 2>(c1, A1, p1);
    mp_mul<5, 4>(c2, A2, p2);
    u32 w[9];
#pragma unroll
    for (int i = 0; i < 9; i++) w[i] = i < 5 ? p1[i] : 0;
    mp_sub<9>(k1, w);
    mp_sub<9>(k1, p2);
    // k2 = c1 |b1| - c2 b2
    u32 k2[9], q1[7], q2[7];
    mp_mul<3, 4>(c1, B1, q1);
    mp_mul<5, 2>(c2, B2, q2);
#pragma unroll
    for (int i = 0; i < 9; i++) { k2[i] = i < 7 ? q1[i] : 0; w[i] = i < 7 ? q2[i] : 0; }
    mp_sub<9>(k2, w);
    GlvScalar r;
    r.neg = (mp_abs<9>(k1) ? 1u : 0u) | (mp_abs<9>(k2) ? 2u : 0u);
#pragma unroll
    for (int i = 0; i < 4; i++) { r.k1[i] = k1[i]; r.k2[i] = k2[i]; }
    r.pad[0] = r.pad[1] = r.pad[2] = 0;
    return r;
}
// glv[i] = decomposition of the canonical scalar tw[i]
__global__ void __launch_bounds__(128) k_glv_decompose(const uint64_t* __restrict__ tw, u32 count, GlvScalar* __restrict__ glv) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) glv[i] = glv_decompose(Fr::load_nc(tw + 4 * (size_t)i));
}
__device__ __forceinline__ Fq fq_beta() {  // beta in Montgomery form
    Fq b;
    b.l[0] = 0xd782e155u; b.l[1] = 0x71930c11u; b.l[2] = 0xffbe3323u; b.l[3] = 0xa6bb947cu;
    b.l[4] = 0xd4741444u; b.l[5] = 0xaa303344u; b.l[6] = 0x26594943u; b.l[7] = 0x2c3b3f0du;
    return b;
}
// s * p = k1 * p + k2 * phi(p): 2-bit joint windows over T[i + 4 j] = i * (+-p) + j * (+-phi(p))
static __device__ __noinline__ XYZZ xyzz_glv_mul(const XYZZ& p, const GlvScalar& s) {
    if (p.is_identity()) return p;
    XYZZ T[16];
    T[0] = XYZZ::identity();
    T[1] = (s.neg & 1u) ? p.neg() : p;
    T[4] = (s.neg & 2u) ? p.neg() : p;
    T[4].x = T[4].x * fq_beta();
    T[2] = xyzz_dbl(T[1]);
    T[3] = T[2];
    xyzz_add(T[3], T[1]);
    T[8] = xyzz_dbl(T[4]);
    T[12] = T[8];
    xyzz_add(T[12], T[4]);
#pragma unroll 1
    for (int j = 1; j < 4; j++)
#pragma unroll 1
        for (int i = 1; i < 4; i++) {
            T[4 * j + i] = T[4 * j];
            xyzz_add(T[4 * j + i], T[i]);
        }
    XYZZ acc = XYZZ::identity();
#pragma unroll 1
    for (int limb = 3; limb >= 0; limb--) {
        u32 v1 = 0, v2 = 0;
#pragma unroll
        for (int t = 0; t < 4; t++)
            if (t == limb) { v1 = s.k1[t]; v2 = s.k2[t]; }
#pragma unroll 1
        for (int sh = 30; sh >= 0; sh -= 2) {
            acc = xyzz_dbl(acc);
            acc = xyzz_dbl(acc);
            const u32 idx = ((v1 >> sh) & 3u) | (((v2 >> sh) & 3u) << 2);
            if (idx) xyzz_add(acc, T[idx]);
        }
    }
    return acc;
}

__device__ __forceinline__ u32 bitrev(u32 x, u32 bits) { return bits ? __brev(x) >> (32 - bits) : 0; }

__global__ void __launch_bounds__(256) k_affine_to_xyzz_bitrev(const Affine* __restrict__ in, u32 k, XYZZ* __restrict__ out) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >> k) return;
    XYZZ::from_affine(Affine::load(in + i)).store(out + bitrev(i, k));
}
// tw[i] = base^i (canonical limbs) for i < count, from pw[j] = base^(2^j)
__global__ void __launch_bounds__(256) k_power_table(const uint64_t* __restrict__ pw, u32 count, int canonical, uint64_t* __restrict__ tw) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Fr r = Fr::one();
    for (u32 j = 0; (i >> j) != 0; j++)
        if ((i >> j) & 1) r = r * Fr::load_nc(pw + 4 * (size_t)j);
    (canonical ? r.from_mont() : r).store(tw + 4 * (size_t)i);
}
// pw[j] = x^(2^j), j < 32;  extra[0] = (2^k)^-1 canonical, extra[1] = (x^(2^k) - 1) / 2^k (Montgomery)
__global__ void k_srs_consts(Fr x, u32 k, uint64_t* __restrict__ pw, uint64_t* __restrict__ extra) {
    if (threadIdx.x | blockIdx.x) return;
    Fr xn = x;
    for (u32 j = 0; j < 32; j++) {
        x.store(pw + 4 * j);
        if (j == k) xn = x;
        x = x.sqr();
    }
    Fr n = Fr::zero();
    n.l[k >> 5] = 1u << (k & 31);
    const Fr n_inv = n.to_mont().inv_bgcd();
    n_inv.from_mont().store(extra);
    ((xn - Fr::one()) * n_inv).store(extra + 4);
}
// stage s (1-based): pairs (i0, i0 + half), twiddle tw[j << (k - s)]
__global__ void __launch_bounds__(128) k_ecfft_stage(XYZZ* __restrict__ pts, const GlvScalar* __restrict__ tw, u32 k, u32 s) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >> (k - 1)) return;
    const u32 half = 1u << (s - 1), j = t & (half - 1), i0 = ((t >> (s - 1)) << s) + j, i1 = i0 + half;
    XYZZ a = XYZZ::load(pts + i0), b = XYZZ::load(pts + i1);
    if (j) b = xyzz_glv_mul(b, tw[(size_t)j << (k - s)]);
    XYZZ lo = a;
    xyzz_add(lo, b);
    xyzz_add(a, b.neg());
    lo.store(pts + i0);
    a.store(pts + i1);
}
__global__ void __launch_bounds__(128) k_scale_to_affine(const XYZZ* __restrict__ pts, const GlvScalar* __restrict__ scalar, u32 n,
                                                         Affine* __restrict__ out) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    xyzz_to_affine(xyzz_glv_mul(XYZZ::load(pts + i), *scalar)).store(out + i);
}
// den[i] = tau - omega^i
__global__ void __launch_bounds__(256) k_lagrange_den(Fr tau, const uint64_t* __restrict__ omega_pows, u32 n, uint64_t* __restrict__ den) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) (tau - Fr::load_nc(omega_pows + 4 * (size_t)i)).store(den + 4 * (size_t)i);
}
// l[i] = c * omega^i * den_inv[i]
__global__ void __launch_bounds__(256) k_lagrange_scalars(const uint64_t* __restrict__ c, const uint64_t* __restrict__ omega_pows,
                                                          const uint64_t* __restrict__ den_inv, u32 n, uint64_t* __restrict__ l) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) (Fr::load_nc(c) * Fr::load_nc(omega_pows + 4 * (size_t)i) * Fr::load_nc(den_inv + 4 * (size_t)i)).store(l + 4 * (size_t)i);
}
__global__ void __launch_bounds__(256) k_on_curve(const Affine* __restrict__ pts, size_t n, u32* __restrict__ bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Affine p = Affine::load(pts + i);
    if (p.is_identity()) return;
    Fq three = Fq::one().dbl() + Fq::one();
    if (!(p.y.sqr() - (p.x.sqr() * p.x + three)).is_zero()) atomicAdd(bad, 1u);
}

static Fr fr_of(const uint64_t x[4]) {
    Fr r;
    memcpy(&r, x, sizeof(Fr));
    return r;
}

void g_to_lagrange_run(h2b_ctx* ctx, const void* d_g, uint32_t k, void* d_g_lagrange) {
    H2B_REQUIRE(k <= 28, "g_to_lagrange: k out of range");
    const size_t n = (size_t)1 << k;
    // workspace: XYZZ points | twiddles (n/2 canonical) | pw (32) | extra (2) | GLV halves of the twiddles (n/2) and of 2^-k
    const size_t tw_cnt = n / 2 + 1;
    char* w = (char*)ctx->get(WS_POOL, n * sizeof(XYZZ) + (tw_cnt + 40) * 32 + (tw_cnt + 1) * sizeof(GlvScalar));
    XYZZ* pts = (XYZZ*)w;
    uint64_t* tw = (uint64_t*)(w + n * sizeof(XYZZ));
    uint64_t* pw = tw + 4 * tw_cnt;
    uint64_t* extra = pw + 4 * 32;
    GlvScalar* glv = (GlvScalar*)(extra + 4 * 8);
    GlvScalar* glv_ninv = glv + tw_cnt;
    H2B_LAUNCH(ctx, k_srs_consts, 1, 32, 0, fr_of(FR_OMEGA_INV[k]), k, pw, extra);
    if (n > 1) {
        H2B_LAUNCH(ctx, k_power_table, ceil_div(n / 2, 256), 256, 0, pw, (u32)(n / 2), 1, tw);
        H2B_LAUNCH(ctx, k_glv_decompose, ceil_div(n / 2, 128), 128, 0, tw, (u32)(n / 2), glv);
    }
    H2B_LAUNCH(ctx, k_glv_decompose, 1, 128, 0, extra, 1u, glv_ninv);  // extra[0] = (2^k)^-1, canonical
    H2B_LAUNCH(ctx, k_affine_to_xyzz_bitrev, ceil_div(n, 256), 256, 0, (const Affine*)d_g, k, pts);
    for (uint32_t s = 1; s <= k; s++) H2B_LAUNCH(ctx, k_ecfft_stage, ceil_div(n / 2, 128), 128, 0, pts, (const GlvScalar*)glv, k, s);
    H2B_LAUNCH(ctx, k_scale_to_affine, ceil_div(n, 128), 128, 0, pts, (const GlvScalar*)glv_ninv, (u32)n, (Affine*)d_g_lagrange);
}

void batch_invert_run(h2b_ctx* ctx, void* d_a, size_t n);
void g1_fixed_base_mul_run(h2b_ctx* ctx, const uint64_t base_xy[8], const void* d_scalars, size_t n, void* d_out);

// g[i] = tau^i * base, g_lagrange[i] = L_i(tau) * base; either output may be null
void srs_setup_run(h2b_ctx* ctx, const uint64_t tau[4], const uint64_t base_xy[8], uint32_t k, void* d_g, void* d_g_lagrange) {
    H2B_REQUIRE(k <= 28, "srs_setup: k out of range");
    const size_t n = (size_t)1 << k;
    // workspace: scalars (n) | omega powers (n) | den (n) | pw_tau (32) | extra (2) | pw_omega (32) | extra2 (2)
    uint64_t* w = (uint64_t*)ctx->get(WS_POOL2, (3 * n + 80) * 32);
    uint64_t *sc = w, *om = w + 4 * n, *den = om + 4 * n, *pw_tau = den + 4 * n, *extra = pw_tau + 4 * 32, *pw_om = extra + 4 * 2,
             *extra2 = pw_om + 4 * 32;
    H2B_LAUNCH(ctx, k_srs_consts, 1, 32, 0, fr_of(tau), k, pw_tau, extra);
    if (d_g) {
        H2B_LAUNCH(ctx, k_power_table, ceil_div(n, 256), 256, 0, pw_tau, (u32)n, 0, sc);
        g1_fixed_base_mul_run(ctx, base_xy, sc, n, d_g);
    }
    if (d_g_lagrange) {
        H2B_LAUNCH(ctx, k_srs_consts, 1, 32, 0, fr_of(FR_OMEGA[k]), k, pw_om, extra2);
        H2B_LAUNCH(ctx, k_power_table, ceil_div(n, 256), 256, 0, pw_om, (u32)n, 0, om);
        H2B_LAUNCH(ctx, k_lagrange_den, ceil_div(n, 256), 256, 0, fr_of(tau), om, (u32)n, den);
        batch_invert_run(ctx, den, n);
        H2B_LAUNCH(ctx, k_lagrange_scalars, ceil_div(n, 256), 256, 0, extra + 4, om, den, (u32)n, sc);
        g1_fixed_base_mul_run(ctx, base_xy, sc, n, d_g_lagrange);
    }
}

// number of points that are neither (0,0) nor on y^2 = x^3 + 3 (synchronises)
size_t g1_count_off_curve_run(h2b_ctx* ctx, const void* d_points, size_t n) {
    if (n == 0) return 0;
    u32* d_bad = (u32*)ctx->get(WS_OUT, 256);
    H2B_CUDA(cudaMemsetAsync(d_bad, 0, 4, ctx->stream));
    H2B_LAUNCH(ctx, k_on_curve, ceil_div(n, 256), 256, 0, (const Affine*)d_points, n, d_bad);
    u32* bounce = (u32*)ctx->get_pinned(0, 4096);
    H2B_CUDA(cudaMemcpyAsync(bounce, d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    return bounce[0];
}

// bytes: n x 32 on the device; returns the number of invalid encodings (synchronises the stream)
size_t g1_decompress_run(h2b_ctx* ctx, const void* d_bytes, size_t n, void* d_out_xy) {
    if (n == 0) return 0;
    unsigned long long* d_cnt = (unsigned long long*)ctx->get(WS_MISC, 8);
    H2B_CUDA(cudaMemsetAsync(d_cnt, 0, 8, ctx->stream));
    H2B_LAUNCH(ctx, k_g1_decompress, ceil_div(n, 128), 128, 0, (const uint8_t*)d_bytes, n, (Affine*)d_out_xy, d_cnt);
    unsigned long long* bounce = (unsigned long long*)ctx->get_pinned(2, 4096);
    H2B_CUDA(cudaMemcpyAsync(bounce, d_cnt, 8, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    return (size_t)bounce[0];
}

// points: n affine Montgomery points on the device -> n x 32 bytes on the device (asynchronous)
void g1_compress_run(h2b_ctx* ctx, const void* d_xy, size_t n, void* d_bytes) {
    if (n == 0) return;
    H2B_LAUNCH(ctx, k_g1_compress, ceil_div(n, 256), 256, 0, (const Affine*)d_xy, n, (uint8_t*)d_bytes);
}

}  // namespace h2b
