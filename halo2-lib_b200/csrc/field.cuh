// field.cuh — BN254 Fq / Fr arithmetic for sm_90a: 254-bit Montgomery (R = 2^256), 8 x 32-bit limbs in registers.
//
// Memory layout is the `[u64;4]` little-endian Montgomery contract halo2-lib exposes
// (halo2-base/src/utils/mod.rs:332-377; halo2curves-axiom 0.7.3 bn256::{Fq,Fr}): on a little-endian
// machine 4 x u64 == 8 x u32, so host arrays are consumed as two 128-bit loads per element.
//
// The multiplier is written for the integer pipe: every (mad.lo.cc, madc.hi.cc) pair on the same
// multiplicands is fused by ptxas into ONE `IMAD.WIDE.U32[.X]` with predicate carry, so a product row is
// 4 wide-MADs for the even limbs of `a` + 4 for the odd limbs.  Even-limb and odd-limb partial products are
// kept in two accumulators whose 64-bit register pairs never move; the Montgomery shift by one limb per
// row is absorbed by swapping the roles of the two accumulators (see mont_mul below).
// 16 IMAD.WIDE + 4 adds per row, 8 rows.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace h2b {

typedef uint32_t u32;
typedef uint64_t u64;

// ---------------------------------------------------------------- carry-chain primitives
// PTX has one carry flag; nvcc never emits .cc instructions itself, and volatile asm statements keep
// their relative order, so chains may be composed from these one-instruction helpers.
#define H2B_ASM_3(name, op)                                                                        \
    __device__ __forceinline__ void name(u32& acc, u32 a, u32 b) {                                 \
        asm volatile(op " %0, %1, %2, %0;" : "+r"(acc) : "r"(a), "r"(b));                       \
    }
H2B_ASM_3(mad_lo_cc, "mad.lo.cc.u32")
H2B_ASM_3(madc_lo_cc, "madc.lo.cc.u32")
H2B_ASM_3(madc_hi_cc, "madc.hi.cc.u32")
H2B_ASM_3(madc_hi, "madc.hi.u32")
#undef H2B_ASM_3
__device__ __forceinline__ void mul_wide(u32& lo, u32& hi, u32 a, u32 b) {
    asm volatile("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, %3;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void add_cc(u32& r, u32 a, u32 b) { asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void addc_cc(u32& r, u32 a, u32 b) { asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void addc(u32& r, u32 a, u32 b) { asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void sub_cc(u32& r, u32 a, u32 b) { asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void subc_cc(u32& r, u32 a, u32 b) { asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void subc(u32& r, u32 a, u32 b) { asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }

// ---------------------------------------------------------------- field parameters (SURVEY.md §8c)
struct FqParams {
    __host__ __device__ static constexpr u32 MOD(int i) {
        constexpr u32 v[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return v[i];
    }
    static constexpr u32 INV = 0xe4866389u;  // -p^-1 mod 2^32
    __host__ __device__ static constexpr u32 ONE(int i) {
        constexpr u32 v[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return v[i];
    }  // R mod p
    __host__ __device__ static constexpr u32 R2(int i) {
        constexpr u32 v[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
        return v[i];
    }
};
struct FrParams {
    __host__ __device__ static constexpr u32 MOD(int i) {
        constexpr u32 v[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return v[i];
    }
    static constexpr u32 INV = 0xefffffffu;  // -r^-1 mod 2^32
    __host__ __device__ static constexpr u32 ONE(int i) {
        constexpr u32 v[8] = {0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return v[i];
    }  // R mod r
    __host__ __device__ static constexpr u32 R2(int i) {
        constexpr u32 v[8] = {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u};
        return v[i];
    }
};

template <class P>
struct __align__(16) Fp {
    u32 l[8];

    __device__ __forceinline__ static Fp zero() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; i++) r.l[i] = 0;
        return r;
    }
    __device__ __forceinline__ static Fp one() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; i++) r.l[i] = P::ONE(i);
        return r;
    }
    __device__ __forceinline__ static Fp r2() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; i++) r.l[i] = P::R2(i);
        return r;
    }
    // two 128-bit loads / stores (pointer must be 16-byte aligned: element stride is 32 B)
    __device__ __forceinline__ static Fp load(const void* p) {
        const uint4* q = reinterpret_cast<const uint4*>(p);
        uint4 a = q[0], b = q[1];
        Fp r;
        r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
        r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
        return r;
    }
    __device__ __forceinline__ static Fp load_nc(const void* p) {  // read-only path
        const uint4* q = reinterpret_cast<const uint4*>(p);
        uint4 a = __ldg(q), b = __ldg(q + 1);
        Fp r;
        r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
        r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
        return r;
    }
    __device__ __forceinline__ void store(void* p) const {
        uint4* q = reinterpret_cast<uint4*>(p);
        q[0] = make_uint4(l[0], l[1], l[2], l[3]);
        q[1] = make_uint4(l[4], l[5], l[6], l[7]);
    }
    __device__ __forceinline__ bool is_zero() const {
        return (l[0] | l[1] | l[2] | l[3] | l[4] | l[5] | l[6] | l[7]) == 0;
    }
    __device__ __forceinline__ bool operator==(const Fp& o) const {
        u32 d = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) d |= l[i] ^ o.l[i];
        return d == 0;
    }

    // r = a - p if a >= p else a   (a < 2p)
    __device__ __forceinline__ static Fp reduce_once(const Fp& a) {
        Fp t;
        u32 borrow;
        sub_cc(t.l[0], a.l[0], P::MOD(0));
#pragma unroll
        for (int i = 1; i < 8; i++) subc_cc(t.l[i], a.l[i], P::MOD(i));
        subc(borrow, 0, 0);  // 0xffffffff if a < p
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; i++) r.l[i] = borrow ? a.l[i] : t.l[i];
        return r;
    }
    __device__ __forceinline__ friend Fp operator+(const Fp& a, const Fp& b) {
        Fp s;
        add_cc(s.l[0], a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < 7; i++) addc_cc(s.l[i], a.l[i], b.l[i]);
        addc(s.l[7], a.l[7], b.l[7]);  // p < 2^254: a + b < 2^255, no carry out
        return reduce_once(s);
    }
    __device__ __forceinline__ friend Fp operator-(const Fp& a, const Fp& b) {
        Fp d;
        u32 borrow;
        sub_cc(d.l[0], a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < 8; i++) subc_cc(d.l[i], a.l[i], b.l[i]);
        subc(borrow, 0, 0);  // all-ones if a < b
        Fp r;
        add_cc(r.l[0], d.l[0], P::MOD(0) & borrow);
#pragma unroll
        for (int i = 1; i < 7; i++) addc_cc(r.l[i], d.l[i], P::MOD(i) & borrow);
        addc(r.l[7], d.l[7], P::MOD(7) & borrow);
        return r;
    }
    __device__ __forceinline__ Fp neg() const { return is_zero() ? *this : (zero() - *this); }
    __device__ __forceinline__ Fp dbl() const { return *this + *this; }

    // Montgomery product a*b*R^-1 mod p, fully reduced.
    //
    // E[k] / O[k] hold the limb at absolute position k of the even-start / odd-start accumulator: partial
    // product a_j*b_i lives at positions (i+j, i+j+1), so for a fixed row i the even-j products tile one
    // accumulator and the odd-j products the other, each as ONE carry chain of 4 wide MADs.  In row i the
    // accumulator whose pairs start at position i ("X") owns the limb the reduction must clear; the other
    // ("Y") still holds one live limb at position i (top half of its consumed lowest pair) which is folded
    // into X[i], the carry of that add entering the Y chain at position i+1 — exactly where it belongs.
    // Bounds: running total < 2p before a row and < 2^288 * 2^(32 i) after the products, so the chains
    // that would carry into position i+9 cannot, and the final sum is < 2p.
    __device__ __forceinline__ friend Fp operator*(const Fp& a, const Fp& b) {
#ifdef H2B_MUL_KARATSUBA  // not the default (see the note at mul_karatsuba): kept for reference only
        return mul_karatsuba(a, b);
#else
        return mul_cios(a, b);
#endif
    }
    __device__ __forceinline__ static Fp mul_cios(const Fp& a, const Fp& b) {
        u32 E[17], O[17];
#pragma unroll
        for (int k = 0; k < 17; k++) { E[k] = 0; O[k] = 0; }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            u32* X = (i & 1) ? O : E;
            u32* Y = (i & 1) ? E : O;
            const u32 bi = b.l[i];
            if (i == 0) {
                // fresh accumulators: plain wide multiplies, no carries
                mul_wide(Y[1], Y[2], a.l[1], bi);
                mul_wide(Y[3], Y[4], a.l[3], bi);
                mul_wide(Y[5], Y[6], a.l[5], bi);
                mul_wide(Y[7], Y[8], a.l[7], bi);
                mul_wide(X[0], X[1], a.l[0], bi);
                mul_wide(X[2], X[3], a.l[2], bi);
                mul_wide(X[4], X[5], a.l[4], bi);
                mul_wide(X[6], X[7], a.l[6], bi);
            } else {
                // chain 1: fold Y's live limb into X[i]; odd-j products into Y at (i+1 .. i+8)
                add_cc(X[i], X[i], Y[i]);
                madc_lo_cc(Y[i + 1], a.l[1], bi); madc_hi_cc(Y[i + 2], a.l[1], bi);
                madc_lo_cc(Y[i + 3], a.l[3], bi); madc_hi_cc(Y[i + 4], a.l[3], bi);
                madc_lo_cc(Y[i + 5], a.l[5], bi); madc_hi_cc(Y[i + 6], a.l[5], bi);
                madc_lo_cc(Y[i + 7], a.l[7], bi); madc_hi(Y[i + 8], a.l[7], bi);
                // chain 2: even-j products into X at (i .. i+7), carry limb X[i+8]
                mad_lo_cc(X[i], a.l[0], bi);      madc_hi_cc(X[i + 1], a.l[0], bi);
                madc_lo_cc(X[i + 2], a.l[2], bi); madc_hi_cc(X[i + 3], a.l[2], bi);
                madc_lo_cc(X[i + 4], a.l[4], bi); madc_hi_cc(X[i + 5], a.l[4], bi);
                madc_lo_cc(X[i + 6], a.l[6], bi); madc_hi_cc(X[i + 7], a.l[6], bi);
                addc(X[i + 8], X[i + 8], 0);
            }
            const u32 m = X[i] * P::INV;
            // chain 3: m * (p1,p3,p5,p7) into Y
            mad_lo_cc(Y[i + 1], m, P::MOD(1));  madc_hi_cc(Y[i + 2], m, P::MOD(1));
            madc_lo_cc(Y[i + 3], m, P::MOD(3)); madc_hi_cc(Y[i + 4], m, P::MOD(3));
            madc_lo_cc(Y[i + 5], m, P::MOD(5)); madc_hi_cc(Y[i + 6], m, P::MOD(5));
            madc_lo_cc(Y[i + 7], m, P::MOD(7)); madc_hi(Y[i + 8], m, P::MOD(7));
            // chain 4: m * (p0,p2,p4,p6) into X; X[i] becomes 0 and is dropped
            mad_lo_cc(X[i], m, P::MOD(0));      madc_hi_cc(X[i + 1], m, P::MOD(0));
            madc_lo_cc(X[i + 2], m, P::MOD(2)); madc_hi_cc(X[i + 3], m, P::MOD(2));
            madc_lo_cc(X[i + 4], m, P::MOD(4)); madc_hi_cc(X[i + 5], m, P::MOD(4));
            madc_lo_cc(X[i + 6], m, P::MOD(6)); madc_hi_cc(X[i + 7], m, P::MOD(6));
            addc(X[i + 8], X[i + 8], 0);
        }
        // both accumulators are live at positions 8..15
        Fp s;
        add_cc(s.l[0], E[8], O[8]);
#pragma unroll
        for (int k = 1; k < 7; k++) addc_cc(s.l[k], E[8 + k], O[8 + k]);
        addc(s.l[7], E[15], O[15]);
        return reduce_once(s);
    }

    // a*b + c*d (Montgomery, fully reduced) with ONE interleaved reduction: 192 wide multiplies instead of 256 for two
    // products.  Same accumulator scheme as mul_cios: row i adds a*b_i and c*d_i before the reduction step clears
    // limb i.  Bounds: after row i the running value is (a*b[0..i] + c*d[0..i] + M_i*p) / 2^(32(i+1)) < 2p + p < 2^256,
    // so the 9-limb windows cannot overflow, and the result (a*b + c*d + M*p)/R < 2p^2/R + p < 1.5p needs one
    // conditional subtraction.  Used for the y coordinate of the group law (r*(Q - X3) - S1*PPP = r*(..) + (p - S1)*PPP).
    __device__ __forceinline__ static Fp mul_add_mul(const Fp& a, const Fp& b, const Fp& c, const Fp& d) {
        u32 E[17], O[17];
#pragma unroll
        for (int k = 0; k < 17; k++) { E[k] = 0; O[k] = 0; }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            u32* X = (i & 1) ? O : E;
            u32* Y = (i & 1) ? E : O;
            const u32 bi = b.l[i], di = d.l[i];
            if (i == 0) {
                mul_wide(Y[1], Y[2], a.l[1], bi);
                mul_wide(Y[3], Y[4], a.l[3], bi);
                mul_wide(Y[5], Y[6], a.l[5], bi);
                mul_wide(Y[7], Y[8], a.l[7], bi);
                mul_wide(X[0], X[1], a.l[0], bi);
                mul_wide(X[2], X[3], a.l[2], bi);
                mul_wide(X[4], X[5], a.l[4], bi);
                mul_wide(X[6], X[7], a.l[6], bi);
            } else {
                add_cc(X[i], X[i], Y[i]);
                madc_lo_cc(Y[i + 1], a.l[1], bi); madc_hi_cc(Y[i + 2], a.l[1], bi);
                madc_lo_cc(Y[i + 3], a.l[3], bi); madc_hi_cc(Y[i + 4], a.l[3], bi);
                madc_lo_cc(Y[i + 5], a.l[5], bi); madc_hi_cc(Y[i + 6], a.l[5], bi);
                madc_lo_cc(Y[i + 7], a.l[7], bi); madc_hi(Y[i + 8], a.l[7], bi);
                mad_lo_cc(X[i], a.l[0], bi);      madc_hi_cc(X[i + 1], a.l[0], bi);
                madc_lo_cc(X[i + 2], a.l[2], bi); madc_hi_cc(X[i + 3], a.l[2], bi);
                madc_lo_cc(X[i + 4], a.l[4], bi); madc_hi_cc(X[i + 5], a.l[4], bi);
                madc_lo_cc(X[i + 6], a.l[6], bi); madc_hi_cc(X[i + 7], a.l[6], bi);
                addc(X[i + 8], X[i + 8], 0);
            }
            // second product of the row: odd-j into Y at (i+1 .. i+8), even-j into X at (i .. i+7) (+ carry limb)
            mad_lo_cc(Y[i + 1], c.l[1], di);  madc_hi_cc(Y[i + 2], c.l[1], di);
            madc_lo_cc(Y[i + 3], c.l[3], di); madc_hi_cc(Y[i + 4], c.l[3], di);
            madc_lo_cc(Y[i + 5], c.l[5], di); madc_hi_cc(Y[i + 6], c.l[5], di);
            madc_lo_cc(Y[i + 7], c.l[7], di); madc_hi(Y[i + 8], c.l[7], di);
            mad_lo_cc(X[i], c.l[0], di);      madc_hi_cc(X[i + 1], c.l[0], di);
            madc_lo_cc(X[i + 2], c.l[2], di); madc_hi_cc(X[i + 3], c.l[2], di);
            madc_lo_cc(X[i + 4], c.l[4], di); madc_hi_cc(X[i + 5], c.l[4], di);
            madc_lo_cc(X[i + 6], c.l[6], di); madc_hi_cc(X[i + 7], c.l[6], di);
            addc(X[i + 8], X[i + 8], 0);
            const u32 m = X[i] * P::INV;
            mad_lo_cc(Y[i + 1], m, P::MOD(1));  madc_hi_cc(Y[i + 2], m, P::MOD(1));
            madc_lo_cc(Y[i + 3], m, P::MOD(3)); madc_hi_cc(Y[i + 4], m, P::MOD(3));
            madc_lo_cc(Y[i + 5], m, P::MOD(5)); madc_hi_cc(Y[i + 6], m, P::MOD(5));
            madc_lo_cc(Y[i + 7], m, P::MOD(7)); madc_hi(Y[i + 8], m, P::MOD(7));
            mad_lo_cc(X[i], m, P::MOD(0));      madc_hi_cc(X[i + 1], m, P::MOD(0));
            madc_lo_cc(X[i + 2], m, P::MOD(2)); madc_hi_cc(X[i + 3], m, P::MOD(2));
            madc_lo_cc(X[i + 4], m, P::MOD(4)); madc_hi_cc(X[i + 5], m, P::MOD(4));
            madc_lo_cc(X[i + 6], m, P::MOD(6)); madc_hi_cc(X[i + 7], m, P::MOD(6));
            addc(X[i + 8], X[i + 8], 0);
        }
        Fp s;
        add_cc(s.l[0], E[8], O[8]);
#pragma unroll
        for (int k = 1; k < 7; k++) addc_cc(s.l[k], E[8 + k], O[8 + k]);
        addc(s.l[7], E[15], O[15]);
        return reduce_once(s);
    }
    // a*b - c*d
    __device__ __forceinline__ static Fp mul_sub_mul(const Fp& a, const Fp& b, const Fp& c, const Fp& d) {
        return mul_add_mul(a, b, c.neg(), d);
    }

    // ---- Karatsuba variant: 48 + 64 = 112 wide multiplies instead of 128 (NOT the default) ------------------------
    // ptxas needs far more instructions for it than for the CIOS form above (incl. IMAD.MOV / IMAD.X on the multiplier
    // pipe), which makes k_accumulate issue- and register-bound; tools/latbench.cu compares the two forms.
    // The idea: the integer multiplier is the scarce resource (plain adds run on the otherwise idle ALU pipe), so one
    // Karatsuba level on the 8x8-limb product
    // trades 16 wide multiplies for ~100 additions:  a = a0 + a1 X, b = b0 + b1 X, X = 2^128,
    //     a*b = z0 + (z0 + z2 - (a0 - a1)(b0 - b1)) X + z2 X^2,   z0 = a0 b0, z2 = a1 b1.
    // 4x4-limb product r[0..8) = x * y.  E / O are position-indexed accumulators for products that start at even /
    // odd limb positions; every chain ends in a carry limb that so far holds only carry counts (see operator*).
    __device__ __forceinline__ static void mul4(const u32* x, const u32* y, u32* r) {
        u32 E[10], O[10];
#pragma unroll
        for (int k = 0; k < 10; k++) { E[k] = 0; O[k] = 0; }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const u32 yi = y[i];
            // products x[j]*y[i] at position i+j; j and j+2 share parity: one carry chain per parity
            u32* A = (i & 1) ? O : E;  // gets j = 0, 2 (positions i, i+2)
            u32* B = (i & 1) ? E : O;  // gets j = 1, 3 (positions i+1, i+3)
            mad_lo_cc(A[i], x[0], yi);      madc_hi_cc(A[i + 1], x[0], yi);
            madc_lo_cc(A[i + 2], x[2], yi); madc_hi_cc(A[i + 3], x[2], yi);
            addc(A[i + 4], A[i + 4], 0);
            mad_lo_cc(B[i + 1], x[1], yi);  madc_hi_cc(B[i + 2], x[1], yi);
            madc_lo_cc(B[i + 3], x[3], yi); madc_hi_cc(B[i + 4], x[3], yi);
            addc(B[i + 5], B[i + 5], 0);
        }
        add_cc(r[0], E[0], O[0]);
#pragma unroll
        for (int k = 1; k < 7; k++) addc_cc(r[k], E[k], O[k]);
        addc(r[7], E[7], O[7]);
    }
    // |x - y| over 4 limbs; returns all-ones if x < y
    __device__ __forceinline__ static u32 absdiff4(const u32* x, const u32* y, u32* d) {
        u32 t[4], borrow;
        sub_cc(t[0], x[0], y[0]);
        subc_cc(t[1], x[1], y[1]);
        subc_cc(t[2], x[2], y[2]);
        subc_cc(t[3], x[3], y[3]);
        subc(borrow, 0, 0);
        // negate when negative: (t ^ borrow) - borrow
        sub_cc(d[0], t[0] ^ borrow, borrow);
        subc_cc(d[1], t[1] ^ borrow, borrow);
        subc_cc(d[2], t[2] ^ borrow, borrow);
        subc(d[3], t[3] ^ borrow, borrow);
        return borrow;
    }
    __device__ __forceinline__ static Fp mul_karatsuba(const Fp& a, const Fp& b) {
        u32 z0[8], z2[8], zm[8], da[4], db[4];
        mul4(a.l, b.l, z0);
        mul4(a.l + 4, b.l + 4, z2);
        const u32 sa = absdiff4(a.l, a.l + 4, da), sb = absdiff4(b.l, b.l + 4, db);
        mul4(da, db, zm);
        // mid = z0 + z2 -+ zm  (9 limbs).  neg = all-ones when (a0-a1)(b0-b1) > 0, i.e. zm is SUBTRACTED
        const u32 neg = ~(sa ^ sb);
        u32 mid[9];
        add_cc(mid[0], z0[0], z2[0]);
#pragma unroll
        for (int k = 1; k < 8; k++) addc_cc(mid[k], z0[k], z2[k]);
        addc(mid[8], 0, 0);
        // mid += (zm ^ neg) + (neg & 1), top limb += neg  (two's complement subtraction when neg)
        add_cc(mid[0], mid[0], neg & 1u);
#pragma unroll
        for (int k = 1; k < 8; k++) addc_cc(mid[k], mid[k], 0);
        addc(mid[8], mid[8], 0);
        add_cc(mid[0], mid[0], zm[0] ^ neg);
#pragma unroll
        for (int k = 1; k < 8; k++) addc_cc(mid[k], mid[k], zm[k] ^ neg);
        addc(mid[8], mid[8], neg);
        // T = z0 + mid * 2^128 + z2 * 2^256  (16 limbs: lo = T[0..8), hi = T[8..16))
        u32 lo[8], hi[8];
#pragma unroll
        for (int k = 0; k < 4; k++) lo[k] = z0[k];
        add_cc(lo[4], z0[4], mid[0]);
        addc_cc(lo[5], z0[5], mid[1]);
        addc_cc(lo[6], z0[6], mid[2]);
        addc_cc(lo[7], z0[7], mid[3]);
        addc_cc(hi[0], z2[0], mid[4]);
        addc_cc(hi[1], z2[1], mid[5]);
        addc_cc(hi[2], z2[2], mid[6]);
        addc_cc(hi[3], z2[3], mid[7]);
        addc_cc(hi[4], z2[4], mid[8]);
        addc_cc(hi[5], z2[5], 0);
        addc_cc(hi[6], z2[6], 0);
        addc(hi[7], z2[7], 0);
        // Montgomery reduction of the low half (8 rows, same even/odd accumulators as operator*), then + hi
        u32 E[17], O[17];
#pragma unroll
        for (int k = 0; k < 17; k++) { E[k] = 0; O[k] = 0; }
#pragma unroll
        for (int k = 0; k < 8; k++) E[k] = lo[k];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            u32* X = (i & 1) ? O : E;
            u32* Y = (i & 1) ? E : O;
            if (i > 0) add_cc(X[i], X[i], Y[i]);  // fold Y's live limb; the carry enters the Y chain below
            const u32 m = X[i] * P::INV;
            if (i > 0) { madc_lo_cc(Y[i + 1], m, P::MOD(1)); } else { mad_lo_cc(Y[i + 1], m, P::MOD(1)); }
            madc_hi_cc(Y[i + 2], m, P::MOD(1));
            madc_lo_cc(Y[i + 3], m, P::MOD(3)); madc_hi_cc(Y[i + 4], m, P::MOD(3));
            madc_lo_cc(Y[i + 5], m, P::MOD(5)); madc_hi_cc(Y[i + 6], m, P::MOD(5));
            madc_lo_cc(Y[i + 7], m, P::MOD(7)); madc_hi(Y[i + 8], m, P::MOD(7));
            mad_lo_cc(X[i], m, P::MOD(0));      madc_hi_cc(X[i + 1], m, P::MOD(0));
            madc_lo_cc(X[i + 2], m, P::MOD(2)); madc_hi_cc(X[i + 3], m, P::MOD(2));
            madc_lo_cc(X[i + 4], m, P::MOD(4)); madc_hi_cc(X[i + 5], m, P::MOD(4));
            madc_lo_cc(X[i + 6], m, P::MOD(6)); madc_hi_cc(X[i + 7], m, P::MOD(6));
            addc(X[i + 8], X[i + 8], 0);
        }
        Fp s;
        add_cc(s.l[0], E[8], O[8]);
#pragma unroll
        for (int k = 1; k < 7; k++) addc_cc(s.l[k], E[8 + k], O[8 + k]);
        addc(s.l[7], E[15], O[15]);
        add_cc(s.l[0], s.l[0], hi[0]);
#pragma unroll
        for (int k = 1; k < 7; k++) addc_cc(s.l[k], s.l[k], hi[k]);
        addc(s.l[7], s.l[7], hi[7]);
        return reduce_once(s);
    }
    // Montgomery square: the same row structure as mul_cios, but row i only multiplies a_i by the limbs j >= i of
    //     a_i, (a_{i+1} << 1), d_{i+2}, ..., d_7        with d = 2a (funnel-shifted limbs),
    // i.e. a_i^2 plus the doubled cross products, each computed once: 36 + 64 = 100 wide multiplies instead of 128.
    // (2 * sum_{j>i} a_j 2^(32j) = sum_{j>i} d_j 2^(32j) minus the top bit of a_i that leaked into d_{i+1}; a < 2^254
    // so d_8 = 0.)  Skipped products of the odd-limb chain still have to pass the carry on: two adds instead of a MAD.
    __device__ __forceinline__ Fp sqr() const {
#ifdef H2B_NO_DEDICATED_SQR
        return (*this) * (*this);
#else
        const Fp& a = *this;
        u32 d[8];
        d[0] = a.l[0] << 1;
#pragma unroll
        for (int j = 1; j < 8; j++) d[j] = __funnelshift_l(a.l[j - 1], a.l[j], 1);
        u32 E[17], O[17];
#pragma unroll
        for (int k = 0; k < 17; k++) { E[k] = 0; O[k] = 0; }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            u32* X = (i & 1) ? O : E;
            u32* Y = (i & 1) ? E : O;
            const u32 bi = a.l[i];
            // multiplier limb j of row i (only used for j >= i)
            auto v = [&](int j) -> u32 { return j == i ? a.l[j] : (j == i + 1 ? (a.l[j] << 1) : d[j]); };
            // chain 1: fold Y's live limb into X[i]; odd-j products (j >= i) into Y at (i+1 .. i+8)
            bool carry_live = false;
            if (i > 0) { add_cc(X[i], X[i], Y[i]); carry_live = true; }
#pragma unroll
            for (int j = 1; j < 8; j += 2) {
                if (j >= i) {
                    if (carry_live) madc_lo_cc(Y[i + j], v(j), bi); else mad_lo_cc(Y[i + j], v(j), bi);
                    if (j == 7) madc_hi(Y[i + j + 1], v(j), bi); else madc_hi_cc(Y[i + j + 1], v(j), bi);
                    carry_live = true;
                } else if (carry_live) {  // skipped product: just pass the carry along
                    addc_cc(Y[i + j], Y[i + j], 0);
                    if (j == 7) addc(Y[i + j + 1], Y[i + j + 1], 0); else addc_cc(Y[i + j + 1], Y[i + j + 1], 0);
                }
            }
            // chain 2: even-j products (j >= i) into X at (i .. i+7), carry limb X[i+8]
            carry_live = false;
#pragma unroll
            for (int j = 0; j < 8; j += 2) {
                if (j >= i) {
                    if (carry_live) madc_lo_cc(X[i + j], v(j), bi); else mad_lo_cc(X[i + j], v(j), bi);
                    madc_hi_cc(X[i + j + 1], v(j), bi);
                    carry_live = true;
                }
            }
            if (carry_live) addc(X[i + 8], X[i + 8], 0);
            const u32 m = X[i] * P::INV;
            mad_lo_cc(Y[i + 1], m, P::MOD(1));  madc_hi_cc(Y[i + 2], m, P::MOD(1));
            madc_lo_cc(Y[i + 3], m, P::MOD(3)); madc_hi_cc(Y[i + 4], m, P::MOD(3));
            madc_lo_cc(Y[i + 5], m, P::MOD(5)); madc_hi_cc(Y[i + 6], m, P::MOD(5));
            madc_lo_cc(Y[i + 7], m, P::MOD(7)); madc_hi(Y[i + 8], m, P::MOD(7));
            mad_lo_cc(X[i], m, P::MOD(0));      madc_hi_cc(X[i + 1], m, P::MOD(0));
            madc_lo_cc(X[i + 2], m, P::MOD(2)); madc_hi_cc(X[i + 3], m, P::MOD(2));
            madc_lo_cc(X[i + 4], m, P::MOD(4)); madc_hi_cc(X[i + 5], m, P::MOD(4));
            madc_lo_cc(X[i + 6], m, P::MOD(6)); madc_hi_cc(X[i + 7], m, P::MOD(6));
            addc(X[i + 8], X[i + 8], 0);
        }
        Fp s;
        add_cc(s.l[0], E[8], O[8]);
#pragma unroll
        for (int k = 1; k < 7; k++) addc_cc(s.l[k], E[8 + k], O[8 + k]);
        addc(s.l[7], E[15], O[15]);
        return reduce_once(s);
#endif
    }

    // Montgomery form -> canonical integer (what `to_repr()` yields; best_multiexp slices these bits)
    __device__ __forceinline__ Fp from_mont() const {
        Fp o = zero();
        o.l[0] = 1;
        return (*this) * o;
    }
    __device__ __forceinline__ Fp to_mont() const { return (*this) * r2(); }

    // a^(p-2); inv(0) = 0.  Cold path (one call per MSM / per batch-inversion block).
    __device__ __noinline__ Fp inv() const {
        Fp acc = one(), base = *this;
#pragma unroll 1
        for (int i = 0; i < 8; i++) {
            u32 e = P::MOD(i);
            if (i == 0) e -= 2;  // MOD[0] >= 2 for both fields: no borrow
#pragma unroll 1
            for (int bit = 0; bit < 32; bit++) {
                if ((e >> bit) & 1) acc = acc * base;
                base = base.sqr();
            }
        }
        return acc;
    }

    // a^-1 by the binary extended Euclidean algorithm: shifts, compares and modular add / sub only, no products.
    // For code where ONE lane inverts while the rest of the CTA waits (k_batch_invert, the small set-up kernels): the
    // Fermat chain above is ~260 dependent squarings = 165 us on a lone warp, this is ~500 halvings + ~250
    // subtractions of 8-limb integers.  Data-dependent branches: do not use it where all lanes invert different values.
    // Invariant: x1 * A = u, x2 * A = v (mod p) with A the value held in the limbs (the Montgomery form aR), so the
    // loop ends with (aR)^-1 as a plain residue; one Montgomery product with R^3 turns that into a^-1 R.  inv(0) = 0.
    __device__ __noinline__ Fp inv_bgcd() const {
        if (is_zero()) return *this;
        Fp u = *this, v, x1 = zero(), x2 = zero();
#pragma unroll
        for (int i = 0; i < 8; i++) v.l[i] = P::MOD(i);
        x1.l[0] = 1;
        auto shr1 = [](Fp& a) {
#pragma unroll
            for (int i = 0; i < 7; i++) a.l[i] = __funnelshift_r(a.l[i], a.l[i + 1], 1);
            a.l[7] >>= 1;
        };
        auto halve = [&](Fp& x) {  // x / 2 mod p: x < p < 2^254, so x + p does not overflow 256 bits
            if (x.l[0] & 1) {
                add_cc(x.l[0], x.l[0], P::MOD(0));
#pragma unroll
                for (int i = 1; i < 7; i++) addc_cc(x.l[i], x.l[i], P::MOD(i));
                addc(x.l[7], x.l[7], P::MOD(7));
            }
            shr1(x);
        };
        auto is_one = [](const Fp& a) { return a.l[0] == 1 && (a.l[1] | a.l[2] | a.l[3] | a.l[4] | a.l[5] | a.l[6] | a.l[7]) == 0; };
        auto sub_if_geq = [](Fp& a, const Fp& b) -> bool {  // a >= b ? (a -= b, true) : false
            Fp d;
            u32 borrow;
            sub_cc(d.l[0], a.l[0], b.l[0]);
#pragma unroll
            for (int i = 1; i < 8; i++) subc_cc(d.l[i], a.l[i], b.l[i]);
            subc(borrow, 0, 0);
            if (borrow) return false;
            a = d;
            return true;
        };
        Fp r;
#pragma unroll 1
        for (;;) {
#pragma unroll 1
            while (!(u.l[0] & 1)) { shr1(u); halve(x1); }
            if (is_one(u)) { r = x1; break; }
#pragma unroll 1
            while (!(v.l[0] & 1)) { shr1(v); halve(x2); }
            if (is_one(v)) { r = x2; break; }
            if (sub_if_geq(u, v)) x1 = x1 - x2;
            else { sub_if_geq(v, u); x2 = x2 - x1; }
        }
        return r * (r2() * r2());  // R^2 * R^2 * R^-1 = R^3;  r * R^3 * R^-1 = r R^2 = a^-1 R
    }

    // ---- a^-1 by constant-time "safegcd" (Bernstein-Yang divsteps; the 30-bit batched form of libsecp256k1's modinv32,
    // restated): 20 rounds of 30 divsteps on the low words build a 2x2 transition matrix that is then applied to the
    // full-width (f, g) and, modulo p, to (d, e) with f = d*A, g = e*A.  No data-dependent branch: every lane of a warp
    // can invert its own element at once, and the work is ~10k add / shift / logic instructions plus ~1800 wide
    // multiplies (the cost of ~15 products) — it runs mostly on the ALU pipe that the Montgomery products leave idle.
    // Used where EVERY thread needs its own inverse (per-thread Montgomery trick in the batch-affine path); the
    // single-lane paths keep inv_bgcd.  inv(0) = 0.  Signed 30-bit limbs: value = sum l[i] 2^(30 i), l[0..7] in [0, 2^30).
    __host__ __device__ static constexpr u32 MOD30(int i) {  // limb i of p in base 2^30
        u64 lo = 0;
        // bits [30 i, 30 i + 30) of the 256-bit modulus
        const int bit = 30 * i, w = bit >> 5, off = bit & 31;
        lo = (u64)(w < 8 ? P::MOD(w) : 0u) | ((u64)(w + 1 < 8 ? P::MOD(w + 1) : 0u) << 32);
        return (u32)((lo >> off) & 0x3fffffffu);
    }
    __host__ __device__ static constexpr u32 MODINV30() {  // p^-1 mod 2^30 (Newton iteration on the low word)
        u32 p0 = P::MOD(0), x = p0;  // x = p^-1 mod 2^3 for odd p
        for (int i = 0; i < 5; i++) x *= 2u - p0 * x;
        return x & 0x3fffffffu;
    }
    __device__ __noinline__ Fp inv_safegcd() const {
        constexpr int32_t M30 = 0x3fffffff;
        int32_t d[9], e[9], f[9], g[9];
        // A (Montgomery limbs, 8 x 32 bits) -> g; p -> f; d = 0, e = 1
        {
            u32 w[9];
#pragma unroll
            for (int i = 0; i < 8; i++) w[i] = l[i];
            w[8] = 0;
#pragma unroll
            for (int i = 0; i < 9; i++) {
                const int bit = 30 * i, wi = bit >> 5, off = bit & 31;
                u64 two = (u64)w[wi] | ((u64)(wi + 1 < 9 ? w[wi + 1] : 0u) << 32);
                g[i] = (int32_t)((two >> off) & 0x3fffffffu);
                f[i] = (int32_t)MOD30(i);
                d[i] = 0;
                e[i] = 0;
            }
            e[0] = 1;
        }
        int32_t zeta = -1;  // -(delta + 1/2), delta = 1/2
#pragma unroll 1
        for (int round = 0; round < 20; round++) {
            // 30 divsteps on the low words
            u32 u = 1, v = 0, q = 0, r = 1;
            u32 ff = (u32)f[0] | ((u32)f[1] << 30), gg = (u32)g[0] | ((u32)g[1] << 30);
#pragma unroll 6
            for (int i = 0; i < 30; i++) {
                u32 c1 = (u32)(zeta >> 31);
                const u32 mask2 = 0u - (gg & 1u);
                const u32 x = (ff ^ c1) - c1, y = (u ^ c1) - c1, z = (v ^ c1) - c1;
                gg += x & mask2;
                q += y & mask2;
                r += z & mask2;
                c1 &= mask2;
                zeta = (int32_t)(((u32)zeta ^ c1) - 1u);
                ff += gg & c1;
                u += q & c1;
                v += r & c1;
                gg >>= 1;
                u <<= 1;
                v <<= 1;
            }
            const int64_t tu = (int32_t)u, tv = (int32_t)v, tq = (int32_t)q, tr = (int32_t)r;
            // (d, e) <- t * (d, e) / 2^30 mod p
            {
                const int32_t sd = d[8] >> 31, se = e[8] >> 31;
                int32_t md = ((int32_t)tu & sd) + ((int32_t)tv & se), me = ((int32_t)tq & sd) + ((int32_t)tr & se);
                int64_t cd = tu * d[0] + tv * e[0], ce = tq * d[0] + tr * e[0];
                md -= (int32_t)((MODINV30() * (u32)cd + (u32)md) & (u32)M30);
                me -= (int32_t)((MODINV30() * (u32)ce + (u32)me) & (u32)M30);
                cd += (int64_t)MOD30(0) * md;
                ce += (int64_t)MOD30(0) * me;
                cd >>= 30;
                ce >>= 30;
#pragma unroll
                for (int i = 1; i < 9; i++) {
                    cd += tu * d[i] + tv * e[i] + (int64_t)MOD30(i) * md;
                    ce += tq * d[i] + tr * e[i] + (int64_t)MOD30(i) * me;
                    d[i - 1] = (int32_t)cd & M30;
                    e[i - 1] = (int32_t)ce & M30;
                    cd >>= 30;
                    ce >>= 30;
                }
                d[8] = (int32_t)cd;
                e[8] = (int32_t)ce;
            }
            // (f, g) <- t * (f, g) / 2^30 (exact)
            {
                int64_t cf = tu * f[0] + tv * g[0], cg = tq * f[0] + tr * g[0];
                cf >>= 30;
                cg >>= 30;
#pragma unroll
                for (int i = 1; i < 9; i++) {
                    cf += tu * f[i] + tv * g[i];
                    cg += tq * f[i] + tr * g[i];
                    f[i - 1] = (int32_t)cf & M30;
                    g[i - 1] = (int32_t)cg & M30;
                    cf >>= 30;
                    cg >>= 30;
                }
                f[8] = (int32_t)cf;
                g[8] = (int32_t)cg;
            }
        }
        // g = 0, f = +-1 (f = p when A = 0, then d = 0): result = sign(f) * d, brought into [0, p)
        // signed limbs -> 288-bit two's complement words
        u32 w[9];
        {
            int64_t acc = 0;
            int have = 0, li = 0;
#pragma unroll
            for (int j = 0; j < 9; j++) {
#pragma unroll
                for (int rep = 0; rep < 3; rep++) {
                    if (have < 32 && li < 9) {
                        acc += (int64_t)((u64)(li < 8 ? (int64_t)d[li] : (int64_t)d[8]) << have);
                        have += 30;
                        li++;
                    }
                }
                w[j] = (u32)acc;
                acc >>= 32;
                have -= 32;
            }
        }
        const u32 negf = (u32)(f[8] >> 31);  // all ones when f = -1
        {   // w <- negf ? -w : w
            u32 c;
            add_cc(w[0], w[0] ^ negf, negf & 1u);
#pragma unroll
            for (int i = 1; i < 8; i++) addc_cc(w[i], w[i] ^ negf, 0);
            addc(w[8], w[8] ^ negf, 0);
            (void)c;
        }
        // w in (-2p, 2p): add p while negative (twice), then subtract p once if >= p
#pragma unroll
        for (int rep = 0; rep < 2; rep++) {
            const u32 neg = (u32)((int32_t)w[8] >> 31);
            add_cc(w[0], w[0], P::MOD(0) & neg);
#pragma unroll
            for (int i = 1; i < 8; i++) addc_cc(w[i], w[i], P::MOD(i) & neg);
            addc(w[8], w[8], 0);
        }
        Fp res;
#pragma unroll
        for (int i = 0; i < 8; i++) res.l[i] = w[i];
        res = reduce_once(res);  // w[8] == 0 now and the value is < 2p
        return res * (r2() * r2());  // plain residue (aR)^-1 -> Montgomery a^-1 R
    }
};

typedef Fp<FqParams> Fq;
typedef Fp<FrParams> Fr;

}  // namespace h2b
