/* oracle/bn254_oracle.c — plain-C CPU restatement of the create_proof hot path (MSM / NTT / assignment).
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * `--impl reference` legs may load the library built from this file.  The product (halo2-lib_b200/)
 * never links, loads or calls it, and has no CPU fallback.
 *
 * PARITY STATUS: **unpinned by reference goldens** — the arithmetic lives in crates that are not
 * vendored under the reference tree and cannot be built here (no Rust toolchain):
 *   halo2curves-axiom 0.7.3 (Cargo.lock:1185-1188)  bn256::{Fq,Fr,G1,G1Affine}, msm::best_multiexp
 *   halo2-axiom 0.5.3 @5e4f0e5 (Cargo.lock:1063-1065) arithmetic::best_fft, poly::EvaluationDomain,
 *                                                      poly::kzg::commitment::ParamsKZG::commit{,_lagrange}
 * and the reference's tests hold no golden vector for them (SURVEY.md §4/§8c).  All outputs are
 * mathematically unique; this file is pinned against oracle/pyref.py (independent Python big-int
 * formulas) and the public alt_bn128 constants / EIP-196 doubling vector in tests/.
 *
 * Each function cites the reference call site / upstream function it restates.
 * Data layout everywhere: field element = uint64_t[4] little-endian limbs, Montgomery form, R = 2^256
 * (the `[u64;4]` contract of halo2-base/src/utils/mod.rs:332-377); G1Affine = x||y (8 limbs),
 * identity = (0,0); G1 (Jacobian) = x||y||z (12 limbs), identity z = 0.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint64_t u64;
typedef unsigned __int128 u128;

typedef struct {
    u64 p[4];    /* modulus */
    u64 inv;     /* -p^{-1} mod 2^64 */
    u64 r2[4];   /* R^2 mod p */
    u64 one[4];  /* R mod p */
} field_t;

/* Constants: SURVEY.md §8(c) (verified with Python in tests/test_oracle_kat.py). */
static const field_t FQ = {
    {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},
    0x87d20782e4866389ULL,
    {0xf32cfc5b538afa89ULL, 0xb5e71911d44501fbULL, 0x47ab1eff0a417ff6ULL, 0x06d89f71cab8351fULL},
    {0xd35d438dc58f0d9dULL, 0x0a78eb28f5c70b3dULL, 0x666ea36f7879462cULL, 0x0e0a77c19a07df2fULL}};
static const field_t FR = {
    {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},
    0xc2e1f593efffffffULL,
    {0x1bb8e645ae216da7ULL, 0x53fe3ab1e35c59e3ULL, 0x8c49833d53bb8085ULL, 0x0216d0b17f4e44a5ULL},
    {0xac96341c4ffffffbULL, 0x36fc76959f60cd29ULL, 0x666ea36f7879462eULL, 0x0e0a77c19a07df2fULL}};

static inline const field_t *F(int which) { return which ? &FR : &FQ; }

/* ------------------------------------------------------------------ field */
static inline int f_is_zero(const u64 a[4]) { return (a[0] | a[1] | a[2] | a[3]) == 0; }
static inline int f_eq(const u64 a[4], const u64 b[4]) {
    return ((a[0] ^ b[0]) | (a[1] ^ b[1]) | (a[2] ^ b[2]) | (a[3] ^ b[3])) == 0;
}
static inline int geq(const u64 a[4], const u64 b[4]) {
    for (int i = 3; i >= 0; i--) {
        if (a[i] > b[i]) return 1;
        if (a[i] < b[i]) return 0;
    }
    return 1;
}
static inline u64 sub4(u64 r[4], const u64 a[4], const u64 b[4]) {
    u64 borrow = 0;
    for (int i = 0; i < 4; i++) {
        u128 t = (u128)a[i] - b[i] - borrow;
        r[i] = (u64)t;
        borrow = (u64)(t >> 64) & 1;
    }
    return borrow;
}
static inline u64 add4(u64 r[4], const u64 a[4], const u64 b[4]) {
    u64 carry = 0;
    for (int i = 0; i < 4; i++) {
        u128 t = (u128)a[i] + b[i] + carry;
        r[i] = (u64)t;
        carry = (u64)(t >> 64);
    }
    return carry;
}
static inline void f_add(const field_t *f, u64 r[4], const u64 a[4], const u64 b[4]) {
    u64 t[4];
    add4(t, a, b); /* p < 2^254: no carry out */
    if (geq(t, f->p)) sub4(r, t, f->p); else memcpy(r, t, 32);
}
static inline void f_sub(const field_t *f, u64 r[4], const u64 a[4], const u64 b[4]) {
    u64 t[4];
    if (sub4(t, a, b)) add4(r, t, f->p); else memcpy(r, t, 32);
}
static inline void f_neg(const field_t *f, u64 r[4], const u64 a[4]) {
    if (f_is_zero(a)) memset(r, 0, 32); else sub4(r, f->p, a);
}
/* Montgomery product, coarsely integrated operand scanning (textbook CIOS). */
static inline void f_mul(const field_t *f, u64 r[4], const u64 a[4], const u64 b[4]) {
    u64 t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
        u64 c = 0;
        for (int j = 0; j < 4; j++) {
            u128 x = (u128)a[j] * b[i] + t[j] + c;
            t[j] = (u64)x;
            c = (u64)(x >> 64);
        }
        u128 y = (u128)t[4] + c;
        t[4] = (u64)y;
        t[5] = (u64)(y >> 64);
        u64 m = t[0] * f->inv;
        u128 x = (u128)m * f->p[0] + t[0];
        c = (u64)(x >> 64);
        for (int j = 1; j < 4; j++) {
            x = (u128)m * f->p[j] + t[j] + c;
            t[j - 1] = (u64)x;
            c = (u64)(x >> 64);
        }
        y = (u128)t[4] + c;
        t[3] = (u64)y;
        t[4] = t[5] + (u64)(y >> 64);
    }
    if (t[4] || geq(t, f->p)) sub4(r, t, f->p); else memcpy(r, t, 32);
}
static inline void f_sqr(const field_t *f, u64 r[4], const u64 a[4]) { f_mul(f, r, a, a); }
static void f_pow(const field_t *f, u64 r[4], const u64 a[4], const u64 e[4]) {
    u64 acc[4], base[4];
    memcpy(acc, f->one, 32);
    memcpy(base, a, 32);
    for (int i = 0; i < 256; i++) {
        if ((e[i >> 6] >> (i & 63)) & 1) f_mul(f, acc, acc, base);
        f_sqr(f, base, base);
    }
    memcpy(r, acc, 32);
}
static void f_inv(const field_t *f, u64 r[4], const u64 a[4]) { /* Fermat; inv(0)=0 */
    u64 e[4], two[4] = {2, 0, 0, 0};
    sub4(e, f->p, two);
    f_pow(f, r, a, e);
}
static inline void f_to_mont(const field_t *f, u64 r[4], const u64 a[4]) { f_mul(f, r, a, f->r2); }
static inline void f_from_mont(const field_t *f, u64 r[4], const u64 a[4]) {
    u64 one[4] = {1, 0, 0, 0};
    f_mul(f, r, a, one);
}

/* exported scalar/batch field ops (tests drive the CUDA field kernels against these) */
void orc_f_mul(int w, const u64 *a, const u64 *b, u64 *r, size_t n) { for (size_t i = 0; i < n; i++) f_mul(F(w), r + 4 * i, a + 4 * i, b + 4 * i); }
void orc_f_add(int w, const u64 *a, const u64 *b, u64 *r, size_t n) { for (size_t i = 0; i < n; i++) f_add(F(w), r + 4 * i, a + 4 * i, b + 4 * i); }
void orc_f_sub(int w, const u64 *a, const u64 *b, u64 *r, size_t n) { for (size_t i = 0; i < n; i++) f_sub(F(w), r + 4 * i, a + 4 * i, b + 4 * i); }
void orc_f_inv(int w, const u64 *a, u64 *r, size_t n) { for (size_t i = 0; i < n; i++) f_inv(F(w), r + 4 * i, a + 4 * i); }
void orc_f_to_mont(int w, const u64 *a, u64 *r, size_t n) { for (size_t i = 0; i < n; i++) f_to_mont(F(w), r + 4 * i, a + 4 * i); }
void orc_f_from_mont(int w, const u64 *a, u64 *r, size_t n) { for (size_t i = 0; i < n; i++) f_from_mont(F(w), r + 4 * i, a + 4 * i); }

/* ------------------------------------------------------------------ G1: y^2 = x^3 + 3, Jacobian */
typedef struct { u64 x[4], y[4], z[4]; } jac_t;
typedef struct { u64 x[4], y[4]; } aff_t;

static inline int aff_is_identity(const aff_t *a) { return f_is_zero(a->x) && f_is_zero(a->y); }
static inline void jac_set_identity(jac_t *r) {
    memset(r, 0, sizeof *r);
    memcpy(r->y, FQ.one, 32); /* halo2curves G1::identity() = (0,1,0) */
}
static inline int jac_is_identity(const jac_t *a) { return f_is_zero(a->z); }

static void jac_double(jac_t *r, const jac_t *p) { /* dbl-2009-l, a = 0 */
    if (jac_is_identity(p)) { jac_set_identity(r); return; }
    const field_t *f = &FQ;
    u64 A[4], B[4], C[4], D[4], E[4], Fv[4], t[4], x3[4], y3[4], z3[4];
    f_sqr(f, A, p->x);
    f_sqr(f, B, p->y);
    f_sqr(f, C, B);
    f_add(f, t, p->x, B); f_sqr(f, t, t); f_sub(f, t, t, A); f_sub(f, t, t, C); f_add(f, D, t, t);
    f_add(f, E, A, A); f_add(f, E, E, A);
    f_sqr(f, Fv, E);
    f_sub(f, x3, Fv, D); f_sub(f, x3, x3, D);
    f_mul(f, z3, p->y, p->z); f_add(f, z3, z3, z3);
    f_sub(f, t, D, x3); f_mul(f, y3, E, t);
    f_add(f, C, C, C); f_add(f, C, C, C); f_add(f, C, C, C);
    f_sub(f, y3, y3, C);
    memcpy(r->x, x3, 32); memcpy(r->y, y3, 32); memcpy(r->z, z3, 32);
}
static void jac_add_mixed(jac_t *r, const jac_t *p, const aff_t *q) { /* madd-2007-bl with special cases */
    const field_t *f = &FQ;
    if (aff_is_identity(q)) { if (r != p) *r = *p; return; }
    if (jac_is_identity(p)) { memcpy(r->x, q->x, 32); memcpy(r->y, q->y, 32); memcpy(r->z, FQ.one, 32); return; }
    u64 z1z1[4], u2[4], s2[4], h[4], rr[4], t[4];
    f_sqr(f, z1z1, p->z);
    f_mul(f, u2, q->x, z1z1);
    f_mul(f, s2, q->y, p->z); f_mul(f, s2, s2, z1z1);
    f_sub(f, h, u2, p->x);
    f_sub(f, rr, s2, p->y);
    if (f_is_zero(h)) {
        if (f_is_zero(rr)) { jac_double(r, p); return; }
        jac_set_identity(r); return;
    }
    u64 hh[4], hhh[4], v[4], x3[4], y3[4], z3[4];
    f_sqr(f, hh, h);
    f_mul(f, hhh, hh, h);
    f_mul(f, v, p->x, hh);
    f_sqr(f, x3, rr); f_sub(f, x3, x3, hhh); f_sub(f, x3, x3, v); f_sub(f, x3, x3, v);
    f_sub(f, t, v, x3); f_mul(f, y3, rr, t); f_mul(f, t, p->y, hhh); f_sub(f, y3, y3, t);
    f_mul(f, z3, p->z, h);
    memcpy(r->x, x3, 32); memcpy(r->y, y3, 32); memcpy(r->z, z3, 32);
}
static void jac_add(jac_t *r, const jac_t *p, const jac_t *q) { /* add-2007-bl style, general */
    const field_t *f = &FQ;
    if (jac_is_identity(q)) { if (r != p) *r = *p; return; }
    if (jac_is_identity(p)) { *r = *q; return; }
    u64 z1z1[4], z2z2[4], u1[4], u2[4], s1[4], s2[4], h[4], rr[4], t[4];
    f_sqr(f, z1z1, p->z); f_sqr(f, z2z2, q->z);
    f_mul(f, u1, p->x, z2z2); f_mul(f, u2, q->x, z1z1);
    f_mul(f, s1, p->y, q->z); f_mul(f, s1, s1, z2z2);
    f_mul(f, s2, q->y, p->z); f_mul(f, s2, s2, z1z1);
    f_sub(f, h, u2, u1); f_sub(f, rr, s2, s1);
    if (f_is_zero(h)) {
        if (f_is_zero(rr)) { jac_double(r, p); return; }
        jac_set_identity(r); return;
    }
    u64 hh[4], hhh[4], v[4], x3[4], y3[4], z3[4];
    f_sqr(f, hh, h); f_mul(f, hhh, hh, h); f_mul(f, v, u1, hh);
    f_sqr(f, x3, rr); f_sub(f, x3, x3, hhh); f_sub(f, x3, x3, v); f_sub(f, x3, x3, v);
    f_sub(f, t, v, x3); f_mul(f, y3, rr, t); f_mul(f, t, s1, hhh); f_sub(f, y3, y3, t);
    f_mul(f, z3, p->z, q->z); f_mul(f, z3, z3, h);
    memcpy(r->x, x3, 32); memcpy(r->y, y3, 32); memcpy(r->z, z3, 32);
}
/* Canonical output form shared with the CUDA side: identity -> (0, R, 0); else (x, y, R) affine-normalised. */
static void jac_normalize(jac_t *p) {
    const field_t *f = &FQ;
    if (jac_is_identity(p)) { jac_set_identity(p); return; }
    u64 zi[4], zi2[4], zi3[4];
    f_inv(f, zi, p->z); f_sqr(f, zi2, zi); f_mul(f, zi3, zi2, zi);
    f_mul(f, p->x, p->x, zi2); f_mul(f, p->y, p->y, zi3); memcpy(p->z, FQ.one, 32);
}

int orc_g1_is_on_curve(const u64 *xy) { /* affine, Montgomery; identity (0,0) counts as on curve */
    const aff_t *a = (const aff_t *)xy;
    if (aff_is_identity(a)) return 1;
    u64 l[4], r[4], three[4] = {3, 0, 0, 0}, b[4];
    f_to_mont(&FQ, b, three);
    f_sqr(&FQ, l, a->y);
    f_sqr(&FQ, r, a->x); f_mul(&FQ, r, r, a->x); f_add(&FQ, r, r, b);
    return f_eq(l, r);
}
void orc_g1_normalize(u64 *xyz) { jac_normalize((jac_t *)xyz); }
void orc_g1_add(const u64 *a, const u64 *b, u64 *out) { /* Jacobian + Jacobian -> normalised */
    jac_t r; jac_add(&r, (const jac_t *)a, (const jac_t *)b); jac_normalize(&r); memcpy(out, &r, 96);
}
/* scalar (Montgomery Fr) * affine base -> normalised Jacobian; plain double-and-add */
static void g1_scalar_mul(jac_t *r, const u64 s_mont[4], const aff_t *b) {
    u64 s[4];
    f_from_mont(&FR, s, s_mont); /* best_multiexp slices `to_repr()` (canonical) bytes: SURVEY.md §3.3 */
    jac_t acc; jac_set_identity(&acc);
    for (int i = 255; i >= 0; i--) {
        jac_double(&acc, &acc);
        if ((s[i >> 6] >> (i & 63)) & 1) jac_add_mixed(&acc, &acc, b);
    }
    *r = acc;
}
void orc_g1_scalar_mul(const u64 *s_mont, const u64 *base_xy, u64 *out) {
    jac_t r; g1_scalar_mul(&r, s_mont, (const aff_t *)base_xy); jac_normalize(&r); memcpy(out, &r, 96);
}
/* out[i] = s_i * base  (affine, normalised; identity -> (0,0)); used to build SRS-like bases */
void orc_g1_fixed_base_mul(const u64 *scalars_mont, size_t n, const u64 *base_xy, u64 *out_xy) {
#pragma omp parallel for schedule(dynamic, 16)
    for (size_t i = 0; i < n; i++) {
        jac_t r; g1_scalar_mul(&r, scalars_mont + 4 * i, (const aff_t *)base_xy);
        if (jac_is_identity(&r)) { memset(out_xy + 8 * i, 0, 64); continue; }
        jac_normalize(&r);
        memcpy(out_xy + 8 * i, r.x, 32); memcpy(out_xy + 8 * i + 4, r.y, 32);
    }
}

/* MSM by definition: sum_i s_i * P_i (what best_multiexp must equal). */
void orc_msm_naive(const u64 *scalars, const u64 *bases, size_t n, u64 *out) {
    jac_t acc; jac_set_identity(&acc);
    for (size_t i = 0; i < n; i++) {
        jac_t t; g1_scalar_mul(&t, scalars + 4 * i, (const aff_t *)(bases + 8 * i));
        jac_add(&acc, &acc, &t);
    }
    jac_normalize(&acc); memcpy(out, &acc, 96);
}

/* Serial Pippenger over one contiguous chunk — the shape of halo2curves `multiexp_serial`
 * (halo2curves-axiom 0.7.3 msm.rs; SURVEY.md App. B): c = 3 (n<32) | ceil(ln n); segments = 256/c + 1;
 * top-down over segments: acc <<= c; (2^c - 1) buckets; digit 0 skipped; running-sum bucket reduction. */
static unsigned get_digit(const u64 s[4], unsigned seg, unsigned c) {
    unsigned bit = seg * c;
    if (bit >= 256) return 0;
    unsigned limb = bit >> 6, off = bit & 63;
    u64 v = s[limb] >> off;
    if (off + c > 64 && limb + 1 < 4) v |= s[limb + 1] << (64 - off);
    return (unsigned)(v & ((1ULL << c) - 1));
}
static void msm_serial(const u64 *canon_scalars, const aff_t *bases, size_t n, jac_t *acc) {
    unsigned c = n < 4 ? 1 : (n < 32 ? 3 : (unsigned)ceil(log((double)n)));
    unsigned segments = 256 / c + 1;
    size_t nb = ((size_t)1 << c) - 1;
    jac_t *buckets = (jac_t *)malloc(nb * sizeof(jac_t));
    jac_set_identity(acc);
    for (int seg = (int)segments - 1; seg >= 0; seg--) {
        for (unsigned i = 0; i < c; i++) jac_double(acc, acc);
        for (size_t b = 0; b < nb; b++) jac_set_identity(&buckets[b]);
        for (size_t i = 0; i < n; i++) {
            unsigned d = get_digit(canon_scalars + 4 * i, (unsigned)seg, c);
            if (d) jac_add_mixed(&buckets[d - 1], &buckets[d - 1], &bases[i]);
        }
        jac_t run; jac_set_identity(&run);
        for (size_t b = nb; b-- > 0;) {
            jac_add(&run, &run, &buckets[b]);
            jac_add(acc, acc, &run);
        }
    }
    free(buckets);
}
/* best_multiexp: split into `threads` contiguous chunks, serial Pippenger each, add partials. */
void orc_msm_pippenger(const u64 *scalars, const u64 *bases, size_t n, int threads, u64 *out) {
    if (threads < 1) threads = 1;
    if ((size_t)threads > n) threads = n ? (int)n : 1;
    u64 *canon = (u64 *)malloc((n ? n : 1) * 32);
#pragma omp parallel for num_threads(threads)
    for (size_t i = 0; i < n; i++) f_from_mont(&FR, canon + 4 * i, scalars + 4 * i);
    jac_t *part = (jac_t *)malloc(threads * sizeof(jac_t));
    size_t chunk = (n + threads - 1) / (threads ? threads : 1);
#pragma omp parallel for num_threads(threads) schedule(static, 1)
    for (int t = 0; t < threads; t++) {
        size_t lo = (size_t)t * chunk, hi = lo + chunk > n ? n : lo + chunk;
        if (lo >= hi) { jac_set_identity(&part[t]); continue; }
        msm_serial(canon + 4 * lo, (const aff_t *)bases + lo, hi - lo, &part[t]);
    }
    jac_t acc; jac_set_identity(&acc);
    for (int t = 0; t < threads; t++) jac_add(&acc, &acc, &part[t]);
    jac_normalize(&acc); memcpy(out, &acc, 96);
    free(part); free(canon);
}

/* ------------------------------------------------------------------ NTT over Fr */
static unsigned bitrev(unsigned x, unsigned bits) {
    unsigned r = 0;
    for (unsigned i = 0; i < bits; i++) { r = (r << 1) | (x & 1); x >>= 1; }
    return r;
}
/* best_fft(a, omega, log_n) (halo2-axiom arithmetic.rs; SURVEY.md App. B): in-place bit reversal,
 * precomputed n/2 twiddles, radix-2 DIT; natural in, natural out: out[i] = sum_j a[j] omega^{ij}. */
void orc_ntt(u64 *a, unsigned log_n, const u64 *omega, int threads) {
    const field_t *f = &FR;
    size_t n = (size_t)1 << log_n;
    if (threads < 1) threads = 1;
    for (size_t i = 0; i < n; i++) {
        size_t j = bitrev((unsigned)i, log_n);
        if (i < j) { u64 t[4]; memcpy(t, a + 4 * i, 32); memcpy(a + 4 * i, a + 4 * j, 32); memcpy(a + 4 * j, t, 32); }
    }
    size_t half_n = n / 2 ? n / 2 : 1;
    u64 *tw = (u64 *)malloc(half_n * 32);
    memcpy(tw, f->one, 32);
    for (size_t i = 1; i < n / 2; i++) f_mul(f, tw + 4 * i, tw + 4 * (i - 1), omega);
    for (unsigned s = 0; s < log_n; s++) {
        size_t half = (size_t)1 << s, step = n / (2 * half);
#pragma omp parallel for num_threads(threads) if (n >= 4096)
        for (size_t b = 0; b < n / 2; b++) {
            size_t grp = b / half, j = b % half;
            u64 *u = a + 4 * (grp * 2 * half + j), *v = u + 4 * half, t[4], x[4];
            f_mul(f, t, v, tw + 4 * (j * step));
            f_sub(f, x, u, t);
            f_add(f, u, u, t);
            memcpy(v, x, 32);
        }
    }
    free(tw);
}
/* serial in-place radix-2 transform with a caller-provided twiddle table tw[i] = root^i, i < n/2 */
static void ntt_serial(u64 *a, unsigned log_n, const u64 *tw) {
    const field_t *f = &FR;
    size_t n = (size_t)1 << log_n;
    for (size_t i = 0; i < n; i++) {
        size_t j = bitrev((unsigned)i, log_n);
        if (i < j) { u64 t[4]; memcpy(t, a + 4 * i, 32); memcpy(a + 4 * i, a + 4 * j, 32); memcpy(a + 4 * j, t, 32); }
    }
    for (unsigned s = 0; s < log_n; s++) {
        size_t half = (size_t)1 << s, step = n / (2 * half);
        for (size_t grp = 0; grp < n; grp += 2 * half)
            for (size_t j = 0; j < half; j++) {
                u64 *u = a + 4 * (grp + j), *v = u + 4 * half, t[4], x[4];
                f_mul(f, t, v, tw + 4 * (j * step));
                f_sub(f, x, u, t);
                f_add(f, u, u, t);
                memcpy(v, x, 32);
            }
    }
}
/* Same contract as orc_ntt, organised for many cores the way a tuned CPU prover would (halo2's best_fft splits the
 * transform into per-thread sub-transforms): n = N1*N2, column transforms + twiddles, row transforms, transpose.
 * Every thread works on whole cache-resident sub-transforms; 3 parallel regions instead of one per butterfly stage.
 * Used for the timed CPU baseline; checked against orc_ntt in tests/test_oracle_kat.py. */
void orc_ntt_fast(u64 *a, unsigned log_n, const u64 *omega, int threads) {
    const field_t *f = &FR;
    if (log_n < 10 || threads <= 1) { orc_ntt(a, log_n, omega, threads); return; }
    unsigned l1 = log_n / 2, l2 = log_n - l1;
    size_t N1 = (size_t)1 << l1, N2 = (size_t)1 << l2, n = N1 * N2;
    /* roots: w1 = omega^N2 (order N1), w2 = omega^N1 (order N2) and their half tables */
    u64 w1[4], w2[4];
    memcpy(w1, omega, 32); for (unsigned i = 0; i < l2; i++) f_sqr(f, w1, w1);
    memcpy(w2, omega, 32); for (unsigned i = 0; i < l1; i++) f_sqr(f, w2, w2);
    u64 *tw1 = (u64 *)malloc((N1 / 2 ? N1 / 2 : 1) * 32), *tw2 = (u64 *)malloc((N2 / 2 ? N2 / 2 : 1) * 32);
    memcpy(tw1, f->one, 32); for (size_t i = 1; i < N1 / 2; i++) f_mul(f, tw1 + 4 * i, tw1 + 4 * (i - 1), w1);
    memcpy(tw2, f->one, 32); for (size_t i = 1; i < N2 / 2; i++) f_mul(f, tw2 + 4 * i, tw2 + 4 * (i - 1), w2);
    u64 *buf = (u64 *)malloc(n * 32);
#pragma omp parallel num_threads(threads)
    {
        u64 *col = (u64 *)malloc(N1 * 32);
        /* step 1+2: for each column j2: N1-point transform over j1 (stride N2), times omega^(j2*i1) */
#pragma omp for schedule(static)
        for (size_t j2 = 0; j2 < N2; j2++) {
            for (size_t j1 = 0; j1 < N1; j1++) memcpy(col + 4 * j1, a + 4 * (j1 * N2 + j2), 32);
            ntt_serial(col, l1, tw1);
            u64 g[4], t[4];
            /* g = omega^j2 */
            memcpy(g, f->one, 32);
            { u64 base[4]; memcpy(base, omega, 32); size_t e = j2; while (e) { if (e & 1) f_mul(f, g, g, base); f_sqr(f, base, base); e >>= 1; } }
            memcpy(t, f->one, 32);
            for (size_t i1 = 0; i1 < N1; i1++) {
                f_mul(f, a + 4 * (i1 * N2 + j2), col + 4 * i1, t);
                f_mul(f, t, t, g);
            }
        }
        /* step 3: rows i1: N2-point transform over j2 (contiguous) */
#pragma omp for schedule(static)
        for (size_t i1 = 0; i1 < N1; i1++) ntt_serial(a + 4 * i1 * N2, l2, tw2);
        /* step 4: out[i1 + N1*i2] = C[i1][i2] */
#pragma omp for schedule(static)
        for (size_t i2 = 0; i2 < N2; i2++)
            for (size_t i1 = 0; i1 < N1; i1++) memcpy(buf + 4 * (i1 + N1 * i2), a + 4 * (i1 * N2 + i2), 32);
        free(col);
    }
    memcpy(a, buf, n * 32);
    free(buf); free(tw1); free(tw2);
}
static int g_fast_ntt = 0; /* orc_use_fast_ntt(1): EvaluationDomain wrappers below go through orc_ntt_fast */
void orc_use_fast_ntt(int on) { g_fast_ntt = on; }
static void ntt_dispatch(u64 *a, unsigned log_n, const u64 *omega, int threads) {
    if (g_fast_ntt) orc_ntt_fast(a, log_n, omega, threads); else orc_ntt(a, log_n, omega, threads);
}
static void fr_from_u64(u64 r[4], u64 v) { u64 t[4] = {v, 0, 0, 0}; f_to_mont(&FR, r, t); }
/* omega of the 2^k domain: ROOT_OF_UNITY^(2^(28-k)); ROOT_OF_UNITY = 7^((r-1)/2^28) (SURVEY.md §8c). */
void orc_omega(unsigned k, u64 *out) {
    u64 g[4], e[4], one[4] = {1, 0, 0, 0};
    fr_from_u64(g, 7);
    sub4(e, FR.p, one);
    /* e = (r-1) >> 28 */
    for (int i = 0; i < 4; i++) e[i] = (e[i] >> 28) | (i < 3 ? e[i + 1] << 36 : 0);
    u64 root[4];
    f_pow(&FR, root, g, e);
    for (unsigned i = k; i < 28; i++) f_sqr(&FR, root, root);
    memcpy(out, root, 32);
}
static void zeta_mont(u64 z[4]) { /* Fr::ZETA = (7^((r-1)/3))^2 ; SURVEY.md §8c */
    static const u64 zc[4] = {0xb8ca0b2d36636f23ULL, 0xcc37a73fec2bc5e9ULL, 0x048b6e193fd84104ULL, 0x30644e72e131a029ULL};
    f_to_mont(&FR, z, zc);
}
/* EvaluationDomain::lagrange_to_coeff: best_fft(omega^-1) then scale by 2^-k */
void orc_lagrange_to_coeff(u64 *a, unsigned k, int threads) {
    u64 w[4], wi[4], n[4], ni[4];
    orc_omega(k, w); f_inv(&FR, wi, w);
    ntt_dispatch(a, k, wi, threads);
    fr_from_u64(n, (u64)1 << k); f_inv(&FR, ni, n);
    size_t N = (size_t)1 << k;
#pragma omp parallel for num_threads(threads) if (N >= 4096)
    for (size_t i = 0; i < N; i++) f_mul(&FR, a + 4 * i, a + 4 * i, ni);
}
/* EvaluationDomain::coeff_to_lagrange == best_fft(omega) */
void orc_coeff_to_lagrange(u64 *a, unsigned k, int threads) {
    u64 w[4]; orc_omega(k, w); ntt_dispatch(a, k, w, threads);
}
/* EvaluationDomain::coeff_to_extended: a[i] *= zeta^(i mod 3); zero-pad to 2^ext_k; best_fft(extended_omega) */
void orc_coeff_to_extended(const u64 *coeffs, size_t n_coeffs, unsigned ext_k, u64 *out, int threads) {
    u64 z[3][4], w[4];
    memcpy(z[0], FR.one, 32); zeta_mont(z[1]); f_sqr(&FR, z[2], z[1]);
    size_t N = (size_t)1 << ext_k;
    memset(out, 0, N * 32);
#pragma omp parallel for num_threads(threads) if (n_coeffs >= 4096)
    for (size_t i = 0; i < n_coeffs; i++) f_mul(&FR, out + 4 * i, coeffs + 4 * i, z[i % 3]);
    orc_omega(ext_k, w); ntt_dispatch(out, ext_k, w, threads);
}
/* EvaluationDomain::extended_to_coeff: best_fft(extended_omega^-1), scale 2^-ext_k, a[i] *= zeta^-(i mod 3);
 * caller truncates to n*(d-1). In place on 2^ext_k elements. */
void orc_extended_to_coeff(u64 *a, unsigned ext_k, int threads) {
    u64 z[3][4];
    orc_lagrange_to_coeff(a, ext_k, threads);
    memcpy(z[0], FR.one, 32); zeta_mont(z[2]); f_sqr(&FR, z[1], z[2]); /* z[1]=zeta^-1=zeta^2, z[2]=zeta^-2=zeta */
    size_t N = (size_t)1 << ext_k;
#pragma omp parallel for num_threads(threads) if (N >= 4096)
    for (size_t i = 0; i < N; i++) f_mul(&FR, a + 4 * i, a + 4 * i, z[i % 3]);
}

/* ------------------------------------------------------------------ witness assignment */
/* assign_witnesses, halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312, literal walk.
 * vcol = concatenation of ctx.advice over threads (Trivial payloads, N x 4 limbs). cols = ncols x 2^k x 4,
 * pre-zeroed here (WitnessCollection starts advice columns at zero). Returns 0, or -1 where Rust would
 * panic (ran out of columns: index out of bounds at :304; no columns but cells present: :279-286). */
int orc_assign_witnesses(const u64 *vcol, size_t N, const u64 *break_points, size_t nbp, unsigned k,
                         size_t ncols, u64 *cols) {
    size_t rows = (size_t)1 << k;
    memset(cols, 0, ncols * rows * 32);
    if (ncols == 0) return N == 0 ? 0 : -1;
    size_t bpi = 0, gate_index = 0, row_offset = 0;
    for (size_t i = 0; i < N; i++) {
        if (row_offset >= rows) return -1;
        memcpy(cols + 4 * (gate_index * rows + row_offset), vcol + 4 * i, 32);
        if (bpi < nbp && break_points[bpi] == row_offset) {
            bpi++;
            row_offset = 0;
            gate_index++;
            if (gate_index >= ncols) return -1;
            memcpy(cols + 4 * (gate_index * rows + row_offset), vcol + 4 * i, 32);
        }
        row_offset++;
    }
    return 0;
}
/* LookupAnyManager::assign_raw, halo2-base/src/virtual_region/lookups.rs:130-155: value j -> col j%L, row j/L */
int orc_assign_lookups(const u64 *vals, size_t N, unsigned k, size_t L, u64 *cols) {
    size_t rows = (size_t)1 << k;
    memset(cols, 0, L * rows * 32);
    if (L == 0) return N == 0 ? 0 : -1;
    for (size_t j = 0; j < N; j++) {
        size_t c = j % L, r = j / L;
        if (r >= rows) return -1;
        memcpy(cols + 4 * (c * rows + r), vals + 4 * j, 32);
    }
    return 0;
}
/* batch_invert_assigned for Rational cells: out = num * den^-1 (den == 0 -> 0), element-wise. */
void orc_eval_rational(const u64 *num, const u64 *den, size_t n, u64 *out) {
    for (size_t i = 0; i < n; i++) {
        u64 di[4]; f_inv(&FR, di, den + 4 * i); f_mul(&FR, out + 4 * i, num + 4 * i, di);
    }
}
/* ff 0.13 BatchInvert::batch_invert semantics on a slice: a[i] <- a[i]^-1, zeros skipped (stay zero);
 * Montgomery's trick exactly as the trait does it (prefix products, one inversion, backward pass). */
void orc_batch_invert(u64 *a, size_t n) {
    u64 *tmp = (u64 *)malloc((n ? n : 1) * 32), acc[4];
    memcpy(acc, FR.one, 32);
    for (size_t i = 0; i < n; i++) {
        memcpy(tmp + 4 * i, acc, 32);
        if (!f_is_zero(a + 4 * i)) f_mul(&FR, acc, acc, a + 4 * i);
    }
    f_inv(&FR, acc, acc);
    for (size_t i = n; i-- > 0;) {
        if (f_is_zero(a + 4 * i)) continue;
        u64 t[4];
        f_mul(&FR, t, acc, tmp + 4 * i);
        f_mul(&FR, acc, acc, a + 4 * i);
        memcpy(a + 4 * i, t, 32);
    }
    free(tmp);
}
/* halo2 permutation / lookup product column (plonk/permutation/prover.rs, plonk/lookup/prover.rs; SURVEY.md §3.3 step 4):
 * z[0] = start; z[row] = z[row-1] * f[row-1] for row in 1..n. */
void orc_grand_product(const u64 *f, const u64 *start, size_t n, u64 *z) {
    if (n == 0) return;
    memcpy(z, start, 32);
    for (size_t row = 1; row < n; row++) f_mul(&FR, z + 4 * row, z + 4 * (row - 1), f + 4 * (row - 1));
}
/* Custom-gate term of halo2-base's vertical gate q*(a + b*c - out), rotations 0..3 of ONE advice column
 * (halo2-base/src/gates/flex_gate/mod.rs:80-91), on the extended domain, folded like halo2's evaluate_h folds gate
 * terms (`value = value * y + gate`): rotation by r rows = index + r * 2^(ext_k - k) mod 2^ext_k. */
void orc_flex_gate_fold(const u64 *q, const u64 *a, const u64 *y, unsigned k, unsigned ext_k, u64 *acc) {
    size_t n = (size_t)1 << ext_k, s = (size_t)1 << (ext_k - k), mask = n - 1;
    for (size_t i = 0; i < n; i++) {
        u64 t[4], g[4];
        f_mul(&FR, t, a + 4 * ((i + s) & mask), a + 4 * ((i + 2 * s) & mask));
        f_add(&FR, t, t, a + 4 * i);
        f_sub(&FR, t, t, a + 4 * ((i + 3 * s) & mask));
        f_mul(&FR, g, q + 4 * i, t);
        f_mul(&FR, t, acc + 4 * i, y);
        f_add(&FR, acc + 4 * i, t, g);
    }
}
/* ---- general quotient evaluation: halo2-axiom 0.5.3 plonk/evaluation.rs (`GraphEvaluator::evaluate`, `Evaluator::evaluate_h`;
 * not vendored — restated from the upstream algorithm; the single gate and lookup halo2-lib feeds it are
 * halo2-base/src/gates/flex_gate/mod.rs:80-91 and gates/range/mod.rs:131-140).  Row loops are written the way the
 * Rust code walks them (running `beta_term`, sequential Horner), not the way the CUDA kernels do. */
typedef struct {
    const uint32_t *program; size_t program_words; uint32_t n_calculations; uint32_t result;
    const u64 *constants; size_t n_constants;
    const int32_t *rotations; size_t n_rotations;
    const u64 *const *fixed; size_t n_fixed;
    const u64 *const *advice; size_t n_advice;
    const u64 *const *instance; size_t n_instance;
    const u64 *challenges; size_t n_challenges;
    u64 beta[4], gamma[4], theta[4], y[4];
} orc_graph; /* same field order as h2b_graph, so tests can pass one ctypes structure to both sides */

static size_t rotation_idx(size_t idx, int rot, unsigned rot_scale_log, size_t isize) { /* get_rotation_idx */
    long long v = (long long)idx + (long long)rot * ((long long)1 << rot_scale_log);
    long long m = (long long)isize;
    v %= m; if (v < 0) v += m;
    return (size_t)v;
}
static void graph_source(const orc_graph *g, uint32_t src, size_t idx, unsigned rs, size_t isize, const u64 *prev, const u64 *inter, u64 out[4]) {
    uint32_t kind = src & 15u, index = (src >> 4) & 0xffffu, slot = src >> 20;
    const u64 *p;
    switch (kind) {
        case 0: p = g->constants + 4 * (size_t)index; break;
        case 1: p = inter + 4 * (size_t)index; break;
        case 2: p = g->fixed[index] + 4 * rotation_idx(idx, g->rotations[slot], rs, isize); break;
        case 3: p = g->advice[index] + 4 * rotation_idx(idx, g->rotations[slot], rs, isize); break;
        case 4: p = g->instance[index] + 4 * rotation_idx(idx, g->rotations[slot], rs, isize); break;
        case 5: p = g->challenges + 4 * (size_t)index; break;
        case 6: p = g->beta; break;
        case 7: p = g->gamma; break;
        case 8: p = g->theta; break;
        case 9: p = g->y; break;
        default: p = prev; break;
    }
    memcpy(out, p, 32);
}
static void graph_row(const orc_graph *g, size_t idx, unsigned rs, size_t isize, const u64 *prev, u64 *inter, u64 out[4]) {
    const uint32_t *pc = g->program;
    for (uint32_t t = 0; t < g->n_calculations; t++) {
        uint32_t op = *pc++;
        u64 a[4], b[4], r[4];
        if (op == 6) { /* Horner(start, parts, factor) */
            graph_source(g, pc[0], idx, rs, isize, prev, inter, r);
            graph_source(g, pc[1], idx, rs, isize, prev, inter, b);
            uint32_t np = pc[2];
            pc += 3;
            for (uint32_t j = 0; j < np; j++) {
                graph_source(g, *pc++, idx, rs, isize, prev, inter, a);
                f_mul(&FR, r, r, b);
                f_add(&FR, r, r, a);
            }
        } else {
            graph_source(g, *pc++, idx, rs, isize, prev, inter, a);
            if (op <= 2) graph_source(g, *pc++, idx, rs, isize, prev, inter, b);
            switch (op) {
                case 0: f_add(&FR, r, a, b); break;
                case 1: f_sub(&FR, r, a, b); break;
                case 2: f_mul(&FR, r, a, b); break;
                case 3: f_mul(&FR, r, a, a); break;
                case 4: f_add(&FR, r, a, a); break;
                case 5: f_neg(&FR, r, a); break;
                default: memcpy(r, a, 32); break;
            }
        }
        memcpy(inter + 4 * (size_t)t, r, 32);
    }
    graph_source(g, g->result, idx, rs, isize, prev, inter, out);
}
void orc_quotient_graph(const orc_graph *g, unsigned k, unsigned ext_k, u64 *values) {
    size_t isize = (size_t)1 << ext_k;
#pragma omp parallel
    {
        u64 *inter = (u64 *)malloc(32 * (size_t)(g->n_calculations + 1));
#pragma omp for schedule(static)
        for (size_t idx = 0; idx < isize; idx++) {
            u64 prev[4], out[4];
            memcpy(prev, values + 4 * idx, 32);
            graph_row(g, idx, ext_k - k, isize, prev, inter, out);
            memcpy(values + 4 * idx, out, 32);
        }
        free(inter);
    }
}
static void fold(u64 *value, const u64 *y, const u64 *term) { /* *value = *value * y + term */
    u64 t[4];
    f_mul(&FR, t, value, y);
    f_add(&FR, value, t, term);
}
void orc_lookup_fold(const orc_graph *g, const u64 *z, const u64 *pin, const u64 *ptab, const u64 *l0, const u64 *l_last,
                     const u64 *l_active, unsigned k, unsigned ext_k, u64 *values) {
    size_t isize = (size_t)1 << ext_k;
    unsigned rs = ext_k - k;
    u64 *inter = (u64 *)malloc(32 * (size_t)(g->n_calculations + 1));
    u64 zero[4] = {0, 0, 0, 0};
    for (size_t idx = 0; idx < isize; idx++) {
        u64 table_value[4], t[4], u[4], w[4], a_minus_s[4];
        graph_row(g, idx, rs, isize, zero, inter, table_value);
        size_t r_next = rotation_idx(idx, 1, rs, isize), r_prev = rotation_idx(idx, -1, rs, isize);
        u64 *value = values + 4 * idx;
        const u64 *zc = z + 4 * idx, *a = pin + 4 * idx, *s = ptab + 4 * idx;
        f_sub(&FR, a_minus_s, a, s);
        f_sub(&FR, t, FR.one, zc); f_mul(&FR, t, t, l0 + 4 * idx); fold(value, g->y, t);                 /* l_0 (1 - z) */
        f_mul(&FR, t, zc, zc); f_sub(&FR, t, t, zc); f_mul(&FR, t, t, l_last + 4 * idx); fold(value, g->y, t); /* l_last (z^2 - z) */
        f_add(&FR, t, a, g->beta); f_add(&FR, u, s, g->gamma); f_mul(&FR, t, t, u); f_mul(&FR, t, z + 4 * r_next, t);
        f_mul(&FR, w, zc, table_value); f_sub(&FR, t, t, w); f_mul(&FR, t, t, l_active + 4 * idx); fold(value, g->y, t);
        f_mul(&FR, t, a_minus_s, l0 + 4 * idx); fold(value, g->y, t);                                    /* l_0 (a' - s') */
        f_sub(&FR, t, a, pin + 4 * r_prev); f_mul(&FR, t, a_minus_s, t); f_mul(&FR, t, t, l_active + 4 * idx); fold(value, g->y, t);
    }
    free(inter);
}
/* Fr::ZETA (cube root of unity) and Fr::DELTA = 7^(2^28), recomputed here from their definitions */
static void delta_mont(u64 d[4]) {
    u64 g[4]; fr_from_u64(g, 7);
    memcpy(d, g, 32);
    for (int i = 0; i < 28; i++) f_mul(&FR, d, d, d);
}
void orc_permutation_fold(const u64 *const *z, size_t n_sets, const u64 *const *columns, const u64 *const *sigma, size_t n_cols,
                          size_t chunk_len, const u64 *l0, const u64 *l_last, const u64 *l_active, const u64 *beta, const u64 *gamma,
                          const u64 *y, unsigned blinding_factors, unsigned k, unsigned ext_k, u64 *values) {
    if (n_sets == 0) return;
    size_t isize = (size_t)1 << ext_k;
    unsigned rs = ext_k - k;
    int last_rotation = -((int)blinding_factors + 1);
    u64 zeta[4], delta[4], ext_omega[4], delta_start[4], beta_term[4];
    zeta_mont(zeta); delta_mont(delta); orc_omega(ext_k, ext_omega);
    f_mul(&FR, delta_start, beta, zeta);
    memcpy(beta_term, FR.one, 32); /* extended_omega^start, start = 0 */
    for (size_t idx = 0; idx < isize; idx++) {
        size_t r_next = rotation_idx(idx, 1, rs, isize), r_last = rotation_idx(idx, last_rotation, rs, isize);
        u64 *value = values + 4 * idx, t[4], u[4];
        const u64 *first = z[0] + 4 * idx, *last = z[n_sets - 1] + 4 * idx;
        f_sub(&FR, t, FR.one, first); f_mul(&FR, t, t, l0 + 4 * idx); fold(value, y, t);
        f_mul(&FR, t, last, last); f_sub(&FR, t, t, last); f_mul(&FR, t, t, l_last + 4 * idx); fold(value, y, t);
        for (size_t s = 1; s < n_sets; s++) {
            f_sub(&FR, t, z[s] + 4 * idx, z[s - 1] + 4 * r_last); f_mul(&FR, t, t, l0 + 4 * idx); fold(value, y, t);
        }
        u64 current_delta[4];
        f_mul(&FR, current_delta, delta_start, beta_term);
        for (size_t s = 0; s < n_sets; s++) {
            size_t c0 = s * chunk_len, c1 = c0 + chunk_len < n_cols ? c0 + chunk_len : n_cols;
            u64 left[4], right[4];
            memcpy(left, z[s] + 4 * r_next, 32);
            for (size_t c = c0; c < c1; c++) {
                f_mul(&FR, t, beta, sigma[c] + 4 * idx); f_add(&FR, t, t, columns[c] + 4 * idx); f_add(&FR, t, t, gamma);
                f_mul(&FR, left, left, t);
            }
            memcpy(right, z[s] + 4 * idx, 32);
            for (size_t c = c0; c < c1; c++) {
                f_add(&FR, u, columns[c] + 4 * idx, current_delta); f_add(&FR, u, u, gamma);
                f_mul(&FR, right, right, u);
                f_mul(&FR, current_delta, current_delta, delta);
            }
            f_sub(&FR, t, left, right); f_mul(&FR, t, t, l_active + 4 * idx); fold(value, y, t);
        }
        f_mul(&FR, beta_term, beta_term, ext_omega);
    }
}
/* ---- keygen-side SRS utilities: halo2-axiom 0.5.3 poly/kzg/commitment.rs `g_to_lagrange` (an FFT over G1 with
 * omega^-1, every point scaled by 2^-k, normalised) and `ParamsKZG::setup` for a given tau (not vendored; restated).
 * The FFT here is the textbook iterative one on Jacobian points with a general scalar multiplication per butterfly. */
static void jac_scalar_mul(jac_t *r, const u64 s_mont[4], const jac_t *p) {
    u64 s[4];
    f_from_mont(&FR, s, s_mont);
    jac_t acc; jac_set_identity(&acc);
    for (int i = 255; i >= 0; i--) {
        jac_double(&acc, &acc);
        if ((s[i >> 6] >> (i & 63)) & 1) jac_add(&acc, &acc, p);
    }
    *r = acc;
}
void orc_g_to_lagrange(const u64 *g_xy, unsigned k, u64 *out_xy) {
    size_t n = (size_t)1 << k;
    jac_t *a = (jac_t *)malloc(n * sizeof(jac_t));
    for (size_t i = 0; i < n; i++) { /* bit-reversed load */
        const aff_t *p = (const aff_t *)(g_xy + 8 * i);
        jac_t *d = a + (k ? bitrev((unsigned)i, k) : 0);
        if (aff_is_identity(p)) { jac_set_identity(d); continue; }
        memcpy(d->x, p->x, 32); memcpy(d->y, p->y, 32); memcpy(d->z, FQ.one, 32);
    }
    u64 w_n[4], w_inv[4];
    orc_omega(k, w_n); f_inv(&FR, w_inv, w_n);
    for (unsigned s = 1; s <= k; s++) {
        size_t m = (size_t)1 << s, half = m >> 1;
        u64 w_m[4]; memcpy(w_m, w_inv, 32);
        for (unsigned i = s; i < k; i++) f_mul(&FR, w_m, w_m, w_m); /* omega^-(n/m) */
#pragma omp parallel for schedule(dynamic, 1)
        for (size_t blk = 0; blk < n; blk += m) {
            u64 w[4]; memcpy(w, FR.one, 32);
            for (size_t j = 0; j < half; j++) {
                jac_t t, neg;
                jac_scalar_mul(&t, w, a + blk + j + half);
                neg = t; f_neg(&FQ, neg.y, t.y);
                jac_add(a + blk + j + half, a + blk + j, &neg);
                jac_add(a + blk + j, a + blk + j, &t);
                f_mul(&FR, w, w, w_m);
            }
        }
    }
    u64 nn[4], n_inv[4];
    fr_from_u64(nn, (u64)n); f_inv(&FR, n_inv, nn);
#pragma omp parallel for schedule(dynamic, 16)
    for (size_t i = 0; i < n; i++) {
        jac_t r; jac_scalar_mul(&r, n_inv, a + i);
        if (jac_is_identity(&r)) { memset(out_xy + 8 * i, 0, 64); continue; }
        jac_normalize(&r);
        memcpy(out_xy + 8 * i, r.x, 32); memcpy(out_xy + 8 * i + 4, r.y, 32);
    }
    free(a);
}
/* g[i] = tau^i * base; g_lagrange[i] = L_i(tau) * base, L_i(tau) = (tau^n - 1)/n * omega^i / (tau - omega^i) */
void orc_srs_setup(const u64 *tau, const u64 *base_xy, unsigned k, u64 *g_xy, u64 *g_lagrange_xy) {
    size_t n = (size_t)1 << k;
    u64 *sc = (u64 *)malloc(n * 32), acc[4], w[4], wi[4], c[4], nn[4], t[4];
    memcpy(acc, FR.one, 32);
    for (size_t i = 0; i < n; i++) { memcpy(sc + 4 * i, acc, 32); f_mul(&FR, acc, acc, tau); } /* acc ends as tau^n */
    if (g_xy) orc_g1_fixed_base_mul(sc, n, base_xy, g_xy);
    if (g_lagrange_xy) {
        f_sub(&FR, c, acc, FR.one); fr_from_u64(nn, (u64)n); f_inv(&FR, nn, nn); f_mul(&FR, c, c, nn);
        orc_omega(k, w); memcpy(wi, FR.one, 32);
        for (size_t i = 0; i < n; i++) {
            f_sub(&FR, t, tau, wi); f_inv(&FR, t, t); f_mul(&FR, t, t, wi); f_mul(&FR, sc + 4 * i, t, c);
            f_mul(&FR, wi, wi, w);
        }
        orc_g1_fixed_base_mul(sc, n, base_xy, g_lagrange_xy);
    }
    free(sc);
}
/* ---- lookup argument: `permute_expression_pair` of plonk/lookup/prover.rs (halo2-axiom 0.5.3 is not vendored), walked the
 * way the Rust code does, in the two variants that exist upstream:
 *   zcash_order = 1  zcash halo2: sort the inputs, count the table values in an ordered map, give every first occurrence
 *                    its own value, then hand the left-over table values (ascending) to the repeated rows popped from the back;
 *   zcash_order = 0  PSE halo2 >= 2023 and the forks derived from it (recalled for halo2-axiom): sort inputs AND table, mark
 *                    first occurrences, then walk the rows front to back with two cursors (distinct inputs / sorted table),
 *                    skipping matched pairs and giving every unfilled row the next table value.
 * Returns 0, or -1 for Error::ConstraintSystemFailure (an input value that the table does not hold).  Only the usable
 * rows [0, 2^k - (blinding_factors + 1)) of the outputs are written. */
static int canon_cmp(const void *a, const void *b) { /* Fr::cmp: canonical value, most significant limb first */
    const u64 *x = (const u64 *)a, *y = (const u64 *)b;
    for (int i = 3; i >= 0; i--) { if (x[i] < y[i]) return -1; if (x[i] > y[i]) return 1; }
    return 0;
}
static int permute_zcash(const u64 *input, const u64 *table, unsigned k, unsigned blinding_factors, u64 *permuted_input,
                         u64 *permuted_table) {
    size_t usable = ((size_t)1 << k) - (blinding_factors + 1);
    u64 *a = (u64 *)malloc(usable * 32), *t = (u64 *)malloc(usable * 32);
    size_t *count = (size_t *)calloc(usable, sizeof(size_t)), *repeated = (size_t *)malloc(usable * sizeof(size_t));
    for (size_t i = 0; i < usable; i++) { f_from_mont(&FR, a + 4 * i, input + 4 * i); f_from_mont(&FR, t + 4 * i, table + 4 * i); }
    qsort(a, usable, 32, canon_cmp); /* permuted_input_expression.sort() */
    qsort(t, usable, 32, canon_cmp);
    /* leftover_table_map: distinct table values (ascending) with their counts */
    size_t n_keys = 0;
    for (size_t i = 0; i < usable; i++) {
        if (n_keys && canon_cmp(t + 4 * (n_keys - 1), t + 4 * i) == 0) { count[n_keys - 1]++; continue; }
        memmove(t + 4 * n_keys, t + 4 * i, 32);
        count[n_keys++] = 1;
    }
    int rc = 0;
    size_t n_rep = 0;
    for (size_t row = 0; row < usable && rc == 0; row++) {
        f_to_mont(&FR, permuted_input + 4 * row, a + 4 * row);
        if (row == 0 || canon_cmp(a + 4 * row, a + 4 * (row - 1)) != 0) {
            memcpy(permuted_table + 4 * row, permuted_input + 4 * row, 32);
            u64 *hit = (u64 *)bsearch(a + 4 * row, t, n_keys, 32, canon_cmp);
            if (!hit || count[(hit - t) / 4] == 0) rc = -1; else count[(hit - t) / 4]--;
        } else {
            repeated[n_rep++] = row;
        }
    }
    for (size_t j = 0; j < n_keys && rc == 0; j++)
        for (size_t c = 0; c < count[j]; c++) {
            if (n_rep == 0) { rc = -1; break; }
            f_to_mont(&FR, permuted_table + 4 * repeated[--n_rep], t + 4 * j);
        }
    if (rc == 0 && n_rep != 0) rc = -1; /* assert!(repeated_input_rows.is_empty()) */
    free(a); free(t); free(count); free(repeated);
    return rc;
}
static int permute_sorted_table(const u64 *input, const u64 *table, unsigned k, unsigned blinding_factors, u64 *permuted_input,
                                u64 *permuted_table) {
    size_t usable = ((size_t)1 << k) - (blinding_factors + 1);
    u64 *a = (u64 *)malloc(usable * 32), *t = (u64 *)malloc(usable * 32), *uniq = (u64 *)malloc(usable * 32);
    unsigned char *filled = (unsigned char *)calloc(usable, 1);
    for (size_t i = 0; i < usable; i++) { f_from_mont(&FR, a + 4 * i, input + 4 * i); f_from_mont(&FR, t + 4 * i, table + 4 * i); }
    qsort(a, usable, 32, canon_cmp); /* permuted_input_expression.sort() */
    qsort(t, usable, 32, canon_cmp); /* sorted_table_coeffs.sort() */
    size_t n_uniq = 0;
    for (size_t row = 0; row < usable; row++) { /* first occurrences: *table_value = Some(*input_value) */
        f_to_mont(&FR, permuted_input + 4 * row, a + 4 * row);
        if (row == 0 || canon_cmp(a + 4 * row, a + 4 * (row - 1)) != 0) {
            memcpy(permuted_table + 4 * row, permuted_input + 4 * row, 32);
            filled[row] = 1;
            memcpy(uniq + 4 * n_uniq++, a + 4 * row, 32);
        }
    }
    int rc = 0;
    size_t iu = 0, it = 0;
    for (size_t row = 0; row < usable && rc == 0; row++) {
        while (iu < n_uniq && it < usable && canon_cmp(uniq + 4 * iu, t + 4 * it) == 0) { iu++; it++; }
        if (!filled[row]) {
            /* a distinct input the table does not hold leaves the cursors stuck: the Rust code would index out of
             * range / build an unsatisfiable column; reported as ConstraintSystemFailure like the zcash walk */
            if (it >= usable || (iu < n_uniq && canon_cmp(uniq + 4 * iu, t + 4 * it) < 0)) { rc = -1; break; }
            f_to_mont(&FR, permuted_table + 4 * row, t + 4 * it);
            it++;
        }
    }
    if (rc == 0) {
        while (iu < n_uniq && it < usable && canon_cmp(uniq + 4 * iu, t + 4 * it) == 0) { iu++; it++; }
        if (iu != n_uniq || it != usable) rc = -1;
    }
    free(a); free(t); free(uniq); free(filled);
    return rc;
}
int orc_permute_expression_pair_ordered(const u64 *input, const u64 *table, unsigned k, unsigned blinding_factors, u64 *permuted_input,
                                        u64 *permuted_table, int zcash_order) {
    return zcash_order ? permute_zcash(input, table, k, blinding_factors, permuted_input, permuted_table)
                       : permute_sorted_table(input, table, k, blinding_factors, permuted_input, permuted_table);
}
int orc_permute_expression_pair(const u64 *input, const u64 *table, unsigned k, unsigned blinding_factors, u64 *permuted_input,
                                u64 *permuted_table) {
    return permute_sorted_table(input, table, k, blinding_factors, permuted_input, permuted_table);
}
/* EvaluationDomain::divide_by_vanishing_poly (halo2-axiom 0.5.3 poly/domain.rs, restated): the table of
 * t(zeta * extended_omega^i) = zeta^n * (extended_omega^n)^i - 1 is built by walking until it repeats, inverted, and
 * applied with period 2^(ext_k - k). */
void orc_divide_by_vanishing_poly(u64 *values, unsigned k, unsigned ext_k) {
    size_t period = (size_t)1 << (ext_k - k), n_ext = (size_t)1 << ext_k;
    u64 orig[4], step[4], cur[4], *t = (u64 *)malloc(period * 32);
    zeta_mont(orig); orc_omega(ext_k, step);
    for (unsigned i = 0; i < k; i++) { f_mul(&FR, orig, orig, orig); f_mul(&FR, step, step, step); }
    memcpy(cur, orig, 32);
    for (size_t j = 0; j < period; j++) {
        f_sub(&FR, t + 4 * j, cur, FR.one);
        f_inv(&FR, t + 4 * j, t + 4 * j);
        f_mul(&FR, cur, cur, step);
    }
    for (size_t i = 0; i < n_ext; i++) f_mul(&FR, values + 4 * i, values + 4 * i, t + 4 * (i % period));
    free(t);
}
/* ---- opening arithmetic: halo2-axiom 0.5.3 arithmetic.rs `eval_polynomial` (Horner) and `kate_division` */
void orc_eval_polynomial(const u64 *coeffs, size_t n, const u64 *x, u64 *out) {
    u64 acc[4] = {0, 0, 0, 0};
    for (size_t i = n; i-- > 0;) { f_mul(&FR, acc, acc, x); f_add(&FR, acc, acc, coeffs + 4 * i); }
    memcpy(out, acc, 32);
}
void orc_kate_division(const u64 *a, size_t n, const u64 *z, u64 *q) { /* b = -z; q_i = a_{i+1} - tmp; tmp = q_i * b */
    u64 b[4], tmp[4] = {0, 0, 0, 0};
    f_neg(&FR, b, z);
    for (size_t i = n - 1; i >= 1; i--) {
        u64 lead[4];
        f_sub(&FR, lead, a + 4 * i, tmp);
        memcpy(q + 4 * (i - 1), lead, 32);
        f_mul(&FR, tmp, lead, b);
    }
}
void orc_poly_lincomb(const u64 *const *polys, const u64 *scalars, size_t m, size_t n, u64 *out) {
    for (size_t i = 0; i < n; i++) {
        u64 acc[4] = {0, 0, 0, 0}, t[4];
        for (size_t j = 0; j < m; j++) { f_mul(&FR, t, polys[j] + 4 * i, scalars + 4 * j); f_add(&FR, acc, acc, t); }
        memcpy(out + 4 * i, acc, 32);
    }
}
void orc_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}
int orc_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
