// params.cu — the host side of halo2-lib's params that is no kernel: the tau `gen_srs` draws and the G2 pair every params
// image carries (halo2-base/src/utils/mod.rs:413-443: `ParamsKZG::setup(k, ChaCha20Rng::from_seed(Default::default()))`).
//   h2b_srs_seeded_tau     rand_chacha `ChaCha20Rng::from_seed(seed)` (20 rounds, 64-bit block counter from 0, stream 0),
//                          64 bytes of `fill_bytes` (the u32 words in order, little-endian), `Fr::random` = from_uniform_bytes:
//                          (lo + hi 2^256) mod r
//   h2b_g2_generator_mul   g2 = the EIP-197 generator of the BN254 twist y^2 = x^3 + 3 / (9 + u) over Fq2 = Fq[u] / (u^2 + 1),
//                          s_g2 = tau g2 by affine double-and-add, in the two encodings of a params image
// A few hundred Fq operations per call; C++, Python and Rust front ends all reach this one copy.  (rand_chacha, halo2curves
// and halo2-axiom are not vendored: the conventions are recalled, DESIGN.md §2.)
#include <cstring>

#include "../../include/h2b200.h"
#pragma GCC visibility push(hidden)
#include "../../include/h2b200_prover.hpp"  // HostFq, HostFr
#pragma GCC visibility pop

namespace {
using h2b::HostFq;
using h2b::HostFr;
using Fq = h2b::Fq;

// ---------------------------------------------------------------- ChaCha20 (RFC 7539 block function, djb's 64-bit counter)
inline uint32_t rotl(uint32_t v, int s) { return (v << s) | (v >> (32 - s)); }
inline void quarter(uint32_t* x, int a, int b, int c, int d) {
    x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16);
    x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12);
    x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8);
    x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7);
}
void chacha20_block(const uint8_t seed[32], uint64_t counter, uint32_t out[16]) {
    uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u};
    for (int i = 0; i < 8; i++)
        s[4 + i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
    s[12] = (uint32_t)counter;
    s[13] = (uint32_t)(counter >> 32);
    s[14] = s[15] = 0;  // stream 0
    uint32_t x[16];
    std::memcpy(x, s, sizeof(x));
    for (int r = 0; r < 10; r++) {
        quarter(x, 0, 4, 8, 12); quarter(x, 1, 5, 9, 13); quarter(x, 2, 6, 10, 14); quarter(x, 3, 7, 11, 15);
        quarter(x, 0, 5, 10, 15); quarter(x, 1, 6, 11, 12); quarter(x, 2, 7, 8, 13); quarter(x, 3, 4, 9, 14);
    }
    for (int i = 0; i < 16; i++) out[i] = x[i] + s[i];
}

// ---------------------------------------------------------------- Fq2 = Fq[u] / (u^2 + 1), Montgomery limbs
struct Fq2 {
    Fq c0{}, c1{};
};
Fq fq_neg(const Fq& a) {
    if (HostFq::is_zero(a)) return a;
    Fq r;
    unsigned __int128 borrow = 0;
    for (int i = 0; i < 4; i++) {
        unsigned __int128 t = (unsigned __int128)h2b::FqHostParams::MOD[i] - a[i] - (uint64_t)borrow;
        r[i] = (uint64_t)t;
        borrow = (t >> 64) & 1;
    }
    return r;
}
Fq fq_sub(const Fq& a, const Fq& b) { return HostFq::add(a, fq_neg(b)); }
Fq fq_canonical(const Fq& a) { return HostFq::mul(a, Fq{1, 0, 0, 0}); }
Fq fq_of(const char* hex) {  // canonical big-endian hex -> Montgomery
    uint64_t c[4] = {0, 0, 0, 0};
    for (const char* p = hex; *p; p++) {
        const uint64_t d = (uint64_t)(*p <= '9' ? *p - '0' : (*p | 0x20) - 'a' + 10);
        for (int i = 3; i > 0; i--) c[i] = (c[i] << 4) | (c[i - 1] >> 60);
        c[0] = (c[0] << 4) | d;
    }
    return HostFq::from_canonical(c);
}
Fq2 f2_add(const Fq2& a, const Fq2& b) { return {HostFq::add(a.c0, b.c0), HostFq::add(a.c1, b.c1)}; }
Fq2 f2_sub(const Fq2& a, const Fq2& b) { return {fq_sub(a.c0, b.c0), fq_sub(a.c1, b.c1)}; }
Fq2 f2_mul(const Fq2& a, const Fq2& b) {
    return {fq_sub(HostFq::mul(a.c0, b.c0), HostFq::mul(a.c1, b.c1)), HostFq::add(HostFq::mul(a.c0, b.c1), HostFq::mul(a.c1, b.c0))};
}
Fq2 f2_inv(const Fq2& a) {  // (c0 - c1 u) / (c0^2 + c1^2)
    const Fq t = HostFq::inv(HostFq::add(HostFq::mul(a.c0, a.c0), HostFq::mul(a.c1, a.c1)));
    return {HostFq::mul(a.c0, t), fq_neg(HostFq::mul(a.c1, t))};
}
bool f2_is_zero(const Fq2& a) { return HostFq::is_zero(a.c0) && HostFq::is_zero(a.c1); }
bool f2_eq(const Fq2& a, const Fq2& b) { return a.c0 == b.c0 && a.c1 == b.c1; }

// ---------------------------------------------------------------- G2 affine, `inf` = the point at infinity
struct G2 {
    Fq2 x, y;
    bool inf = false;
};
G2 g2_add(const G2& a, const G2& b) {
    if (a.inf) return b;
    if (b.inf) return a;
    Fq2 lam;
    if (f2_eq(a.x, b.x)) {
        if (f2_is_zero(f2_add(a.y, b.y))) return G2{{}, {}, true};
        const Fq2 xx = f2_mul(a.x, a.x);
        lam = f2_mul(f2_add(f2_add(xx, xx), xx), f2_inv(f2_add(a.y, a.y)));
    } else {
        lam = f2_mul(f2_sub(b.y, a.y), f2_inv(f2_sub(b.x, a.x)));
    }
    const Fq2 x3 = f2_sub(f2_sub(f2_mul(lam, lam), a.x), b.x);
    return G2{x3, f2_sub(f2_mul(lam, f2_sub(a.x, x3)), a.y), false};
}
G2 g2_generator() {  // EIP-197: x = x0 + x1 u, y = y0 + y1 u
    return G2{{fq_of("1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed"),
               fq_of("198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2")},
              {fq_of("12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa"),
               fq_of("090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b")},
              false};
}
G2 g2_mul(const Fq& scalar_canonical, const G2& p) {
    G2 acc{{}, {}, true};
    for (int limb = 3; limb >= 0; limb--)
        for (int bit = 63; bit >= 0; bit--) {
            acc = g2_add(acc, acc);
            if ((scalar_canonical[limb] >> bit) & 1) acc = g2_add(acc, p);
        }
    return acc;
}
// SerdeFormat::Processed: x.c0 | x.c1 canonical little-endian; byte 63 bit 7 = identity, bit 6 = sgn0(y) (the parity of the
// canonical y.c0, or of y.c1 when y.c0 = 0)
void g2_processed(const G2& p, uint8_t out[64]) {
    std::memset(out, 0, 64);
    if (p.inf) {
        out[63] = 0x80;
        return;
    }
    const Fq x0 = fq_canonical(p.x.c0), x1 = fq_canonical(p.x.c1), y0 = fq_canonical(p.y.c0), y1 = fq_canonical(p.y.c1);
    std::memcpy(out, x0.data(), 32);
    std::memcpy(out + 32, x1.data(), 32);
    const bool sign = HostFq::is_zero(y0) ? (y1[0] & 1) : (y0[0] & 1);
    out[63] |= (uint8_t)(sign << 6);
}
// SerdeFormat::RawBytes: x.c0 | x.c1 | y.c0 | y.c1, Montgomery limbs (the identity (0, 0))
void g2_raw(const G2& p, uint8_t out[128]) {
    std::memset(out, 0, 128);
    if (p.inf) return;
    std::memcpy(out, p.x.c0.data(), 32);
    std::memcpy(out + 32, p.x.c1.data(), 32);
    std::memcpy(out + 64, p.y.c0.data(), 32);
    std::memcpy(out + 96, p.y.c1.data(), 32);
}
bool below_r(const uint64_t t[4]) { return !HostFr::geq_mod(t); }
}  // namespace

extern "C" int h2b_srs_seeded_tau(const uint8_t seed[32], uint64_t tau[4]) {
    if (!seed || !tau) return H2B_ERR_ARG;
    uint32_t w[16];
    chacha20_block(seed, 0, w);
    uint8_t bytes[64];
    for (int i = 0; i < 16; i++)
        for (int j = 0; j < 4; j++) bytes[4 * i + j] = (uint8_t)(w[i] >> (8 * j));
    const h2b::Fr t = HostFr::from_wide_bytes(bytes);
    std::memcpy(tau, t.data(), 32);
    return H2B_OK;
}

extern "C" int h2b_g2_generator_mul(const uint64_t tau[4], uint8_t processed[128], uint8_t raw[256]) {
    if (!tau || !below_r(tau)) return H2B_ERR_ARG;
    const G2 g2 = g2_generator();
    const G2 s_g2 = g2_mul(HostFr::mul({tau[0], tau[1], tau[2], tau[3]}, h2b::Fr{1, 0, 0, 0}), g2);
    if (processed) {
        g2_processed(g2, processed);
        g2_processed(s_g2, processed + 64);
    }
    if (raw) {
        g2_raw(g2, raw);
        g2_raw(s_g2, raw + 128);
    }
    return H2B_OK;
}
