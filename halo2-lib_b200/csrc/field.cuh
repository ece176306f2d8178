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
        return mul_cios(a, b);
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

    // Montgomery square: the same row structure as mul_cios, but row i only multiplies a_i by the limbs j >= i of
    //     a_i, (a_{i+1} << 1), d_{i+2}, ..., d_7        with d = 2a (funnel-shifted limbs),
    // i.e. a_i^2 plus the doubled cross products, each computed once: 36 + 64 = 100 wide multiplies instead of 128.
    // (2 * sum_{j>i} a_j 2^(32j) = sum_{j>i} d_j 2^(32j) minus the top bit of a_i that leaked into d_{i+1}; a < 2^254
    // so d_8 = 0.)  Skipped products of the odd-limb chain still have to pass the carry on: two adds instead of a MAD.
    __device__ __forceinline__ Fp sqr() const {
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
};

typedef Fp<FqParams> Fq;
typedef Fp<FrParams> Fr;

}  // namespace h2b
