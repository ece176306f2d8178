// h2b200_prover.hpp — C++ host side of the RESIDENT prover: the data flow of halo2-axiom 0.5.3 `create_proof`
// (sole halo2-lib call site: halo2-base/src/utils/testing.rs:40-48) for the constraint system halo2-base builds, with
// every column kept in HBM behind `h2b_poly` handles between the phases.  It is the one implementation of the proof
// sequence: halo2-lib_b200/prover.py binds it through halo2-lib_b200/csrc/prover_binding.cu, and it is the shape a Rust
// `create_proof` over include/h2b200.h would take (INTEGRATION.md §3b).
//
// Circuit shape (halo2-base `BaseCircuitParams`): A gate-advice columns a0..a{A-1} with selectors q{j} and the vertical
// gate q (a0 + a1 a2 - a3) (flex_gate/mod.rs:80-91); L lookup-advice columns l0..l{L-1} looked up in `table` as they are
// (range/mod.rs:131-150), or with L = 0 the selector lookup q_lookup * a0 (range/mod.rs:92-94), or no lookup; F constants
// columns c, c1..c{F-1} (num_fixed, flex_gate/mod.rs:123-129; F = 0 when the builder uses no constants); I instance columns
// i0..i{I-1} (BaseConfig::configure, gates/circuit/mod.rs:87-93); equality on [c, c1.., a0.., l0.., i0..].
// Degree 5 / 4 / 3, permutation sets of degree - 2 columns, degree - 1 pieces of h.  Instance columns are not committed, blinded
// or opened (KZG: QUERY_INSTANCE = false): their values enter the transcript and the permutation argument only.
//
// The host does what the Rust side does: the Blake2b transcript, the challenges, the blinding scalars and a handful of
// 254-bit modular operations on them (`HostFr`); no polynomial arithmetic happens here.
#pragma once
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <utility>

#include "h2b200.hpp"
#include "h2b200_selectors.hpp"

namespace h2b {

// ------------------------------------------------------------------------------------------------ host-side fields (Montgomery)
// a few dozen multiplications per proof: challenges, rotations of the evaluation point, powers of v and mu (Fr); one
// inversion per downloaded batch of commitments to bring them to affine form before they enter the transcript (Fq) — what
// the Rust side does on the CPU
struct FrHostParams {
    static constexpr uint64_t MOD[4] = {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
    static constexpr uint64_t R1[4] = {0xac96341c4ffffffbULL, 0x36fc76959f60cd29ULL, 0x666ea36f7879462eULL, 0x0e0a77c19a07df2fULL};
    static constexpr uint64_t R2[4] = {0x1bb8e645ae216da7ULL, 0x53fe3ab1e35c59e3ULL, 0x8c49833d53bb8085ULL, 0x0216d0b17f4e44a5ULL};
    static constexpr uint64_t INV = 0xc2e1f593efffffffULL;  // -r^-1 mod 2^64
};
struct FqHostParams {
    static constexpr uint64_t MOD[4] = {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
    static constexpr uint64_t R1[4] = {0xd35d438dc58f0d9dULL, 0x0a78eb28f5c70b3dULL, 0x666ea36f7879462cULL, 0x0e0a77c19a07df2fULL};
    static constexpr uint64_t R2[4] = {0xf32cfc5b538afa89ULL, 0xb5e71911d44501fbULL, 0x47ab1eff0a417ff6ULL, 0x06d89f71cab8351fULL};
    static constexpr uint64_t INV = 0x87d20782e4866389ULL;  // -p^-1 mod 2^64
};
template <class P>
struct HostField {
    using E = std::array<uint64_t, 4>;
    static E one() { return {P::R1[0], P::R1[1], P::R1[2], P::R1[3]}; }
    static bool is_zero(const E& a) { return (a[0] | a[1] | a[2] | a[3]) == 0; }
    static bool geq_mod(const uint64_t a[4]) {
        for (int i = 3; i >= 0; i--) {
            if (a[i] != P::MOD[i]) return a[i] > P::MOD[i];
        }
        return true;
    }
    static void sub_mod(uint64_t a[4]) {
        unsigned __int128 borrow = 0;
        for (int i = 0; i < 4; i++) {
            unsigned __int128 t = (unsigned __int128)a[i] - P::MOD[i] - (uint64_t)borrow;
            a[i] = (uint64_t)t;
            borrow = (t >> 64) & 1;
        }
    }
    static E mul(const E& a, const E& b) {  // Montgomery product (CIOS)
        uint64_t t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 4; i++) {
            unsigned __int128 carry = 0;
            for (int j = 0; j < 4; j++) {
                unsigned __int128 cur = (unsigned __int128)a[j] * b[i] + t[j] + (uint64_t)carry;
                t[j] = (uint64_t)cur;
                carry = cur >> 64;
            }
            unsigned __int128 cur = (unsigned __int128)t[4] + (uint64_t)carry;
            t[4] = (uint64_t)cur;
            t[5] = (uint64_t)(cur >> 64);
            const uint64_t m = t[0] * P::INV;
            carry = ((unsigned __int128)m * P::MOD[0] + t[0]) >> 64;
            for (int j = 1; j < 4; j++) {
                cur = (unsigned __int128)m * P::MOD[j] + t[j] + (uint64_t)carry;
                t[j - 1] = (uint64_t)cur;
                carry = cur >> 64;
            }
            cur = (unsigned __int128)t[4] + (uint64_t)carry;
            t[3] = (uint64_t)cur;
            t[4] = t[5] + (uint64_t)(cur >> 64);
        }
        uint64_t r[4] = {t[0], t[1], t[2], t[3]};
        if (t[4] || geq_mod(r)) sub_mod(r);
        return {r[0], r[1], r[2], r[3]};
    }
    static E add(const E& a, const E& b) {
        uint64_t r[4];
        unsigned __int128 carry = 0;
        for (int i = 0; i < 4; i++) {
            unsigned __int128 t = (unsigned __int128)a[i] + b[i] + (uint64_t)carry;
            r[i] = (uint64_t)t;
            carry = t >> 64;
        }
        if (carry || geq_mod(r)) sub_mod(r);
        return {r[0], r[1], r[2], r[3]};
    }
    static E neg(const E& a) {
        if (is_zero(a)) return a;
        uint64_t r[4] = {P::MOD[0], P::MOD[1], P::MOD[2], P::MOD[3]};
        unsigned __int128 borrow = 0;
        for (int i = 0; i < 4; i++) {
            unsigned __int128 t = (unsigned __int128)r[i] - a[i] - (uint64_t)borrow;
            r[i] = (uint64_t)t;
            borrow = (t >> 64) & 1;
        }
        return {r[0], r[1], r[2], r[3]};
    }
    static E sub(const E& a, const E& b) { return add(a, neg(b)); }
    static E to_canonical(const E& a) { return mul(a, {1, 0, 0, 0}); }  // a R^-1: the value itself, little-endian limbs
    static E from_canonical(const uint64_t c[4]) { return mul({c[0], c[1], c[2], c[3]}, {P::R2[0], P::R2[1], P::R2[2], P::R2[3]}); }
    static E pow(E base, uint64_t e) {
        E acc = one();
        while (e) {
            if (e & 1) acc = mul(acc, base);
            base = mul(base, base);
            e >>= 1;
        }
        return acc;
    }
    static E inv(const E& a) {  // a^(modulus - 2): Fermat, ~380 products (tens of microseconds on the host)
        uint64_t e[4] = {P::MOD[0] - 2, P::MOD[1], P::MOD[2], P::MOD[3]};  // the low limbs of both moduli are >= 2
        E acc = one();
        for (int limb = 3; limb >= 0; limb--)
            for (int bit = 63; bit >= 0; bit--) {
                acc = mul(acc, acc);
                if ((e[limb] >> bit) & 1) acc = mul(acc, a);
            }
        return acc;
    }
};
using HostFq = HostField<FqHostParams>;
struct HostFr : HostField<FrHostParams> {
    // 2^28-th root of unity 7^((r - 1) >> 28), canonical (halo2curves bn256::Fr::ROOT_OF_UNITY)
    static constexpr uint64_t ROOT28[4] = {0xd34f1ed960c37c9cULL, 0x3215cf6dd39329c8ULL, 0x98865ea93dd31f74ULL, 0x03ddb9f5166d18b7ULL};
    // 64 little-endian bytes -> the integer mod r, Montgomery form (the transcript's challenge)
    static Fr from_wide_bytes(const uint8_t d[64]) {
        uint64_t l[4], h[4];
        std::memcpy(l, d, 32);
        std::memcpy(h, d + 32, 32);
        // value = lo + hi 2^256:  mont(lo) = mul(lo, R2),  mont(hi 2^256) = mul(mul(hi, R2), R2)
        const Fr r2 = {FrHostParams::R2[0], FrHostParams::R2[1], FrHostParams::R2[2], FrHostParams::R2[3]};
        while (geq_mod(l)) sub_mod(l);  // Montgomery multiplication wants operands < r
        while (geq_mod(h)) sub_mod(h);
        return add(mul({l[0], l[1], l[2], l[3]}, r2), mul(mul({h[0], h[1], h[2], h[3]}, r2), r2));
    }
    static Fr omega(uint32_t k) {  // generator of the 2^k domain
        Fr w = from_canonical(ROOT28);
        for (uint32_t i = k; i < 28; i++) w = mul(w, w);
        return w;
    }
};
// Jacobian (X, Y, Z) -> (X / Z^2, Y / Z^3, 1), the identity -> all zero: the form in which a commitment enters the transcript
// and the proof (the accumulation order inside an MSM is not deterministic, the Jacobian representative therefore is not either).
// In place over the m commitments of one download with ONE inversion (Montgomery's trick): the host does this between phases
// while the GPU waits.
inline void g1_normalize_host_batch(G1* pts, size_t m) {
    std::vector<Fq> pref(m);  // prefix products over the non-zero z
    Fq acc = HostFq::one();
    for (size_t i = 0; i < m; i++) {
        pref[i] = acc;
        if (!HostFq::is_zero(pts[i].z)) acc = HostFq::mul(acc, pts[i].z);
    }
    Fq inv = HostFq::inv(acc);
    for (size_t i = m; i-- > 0;) {
        G1& p = pts[i];
        if (HostFq::is_zero(p.z)) {
            p = G1{};
            continue;
        }
        const Fq zi = HostFq::mul(inv, pref[i]), zi2 = HostFq::mul(zi, zi);
        inv = HostFq::mul(inv, p.z);
        p = G1{HostFq::mul(p.x, zi2), HostFq::mul(p.y, HostFq::mul(zi2, zi)), HostFq::one()};
    }
}
inline G1 g1_normalize_host(const G1& p) {
    G1 q = p;
    g1_normalize_host_batch(&q, 1);
    return q;
}

// ------------------------------------------------------------------------------------------------ Blake2b-512 (RFC 7693)
class Blake2b {
public:
    Blake2b() {
        for (int i = 0; i < 8; i++) h_[i] = IV[i];
        h_[0] ^= 0x01010000ULL ^ 64;  // digest length 64, no key
    }
    // the same with the 16-byte personalization of the parameter block (bytes 48..63, i.e. h[6], h[7])
    explicit Blake2b(const uint8_t personal[16]) : Blake2b() {
        uint64_t p[2];
        std::memcpy(p, personal, 16);
        h_[6] ^= p[0];
        h_[7] ^= p[1];
    }
    void update(const void* data, size_t len) {
        const uint8_t* p = static_cast<const uint8_t*>(data);
        while (len) {
            if (fill_ == 128) {  // the buffer is only compressed when more input follows (the last block is final)
                t_ += 128;
                compress(false);
                fill_ = 0;
            }
            const size_t take = std::min(len, size_t(128) - fill_);
            std::memcpy(buf_ + fill_, p, take);
            fill_ += take;
            p += take;
            len -= take;
        }
    }
    // digest of everything absorbed so far; the state is left untouched (as hashlib's digest())
    std::array<uint8_t, 64> digest() const {
        Blake2b c = *this;
        c.t_ += c.fill_;
        std::memset(c.buf_ + c.fill_, 0, 128 - c.fill_);
        c.compress(true);
        std::array<uint8_t, 64> out;
        std::memcpy(out.data(), c.h_, 64);
        return out;
    }

private:
    static constexpr uint64_t IV[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                       0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
    static uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
    void compress(bool last) {
        static const uint8_t S[12][16] = {
            {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
            {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
            {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
            {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
            {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
            {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
        uint64_t m[16], v[16];
        std::memcpy(m, buf_, 128);
        for (int i = 0; i < 8; i++) { v[i] = h_[i]; v[i + 8] = IV[i]; }
        v[12] ^= t_;
        if (last) v[14] = ~v[14];
        auto G = [&](int a, int b, int c, int d, uint64_t x, uint64_t y) {
            v[a] = v[a] + v[b] + x; v[d] = rotr(v[d] ^ v[a], 32);
            v[c] = v[c] + v[d];     v[b] = rotr(v[b] ^ v[c], 24);
            v[a] = v[a] + v[b] + y; v[d] = rotr(v[d] ^ v[a], 16);
            v[c] = v[c] + v[d];     v[b] = rotr(v[b] ^ v[c], 63);
        };
        for (int r = 0; r < 12; r++) {
            const uint8_t* s = S[r];
            G(0, 4, 8, 12, m[s[0]], m[s[1]]);   G(1, 5, 9, 13, m[s[2]], m[s[3]]);
            G(2, 6, 10, 14, m[s[4]], m[s[5]]);  G(3, 7, 11, 15, m[s[6]], m[s[7]]);
            G(0, 5, 10, 15, m[s[8]], m[s[9]]);  G(1, 6, 11, 12, m[s[10]], m[s[11]]);
            G(2, 7, 8, 13, m[s[12]], m[s[13]]); G(3, 4, 9, 14, m[s[14]], m[s[15]]);
        }
        for (int i = 0; i < 8; i++) h_[i] ^= v[i] ^ v[i + 8];
    }
    uint64_t h_[8];
    uint64_t t_ = 0;
    uint8_t buf_[128] = {};
    size_t fill_ = 0;
};

// Blake2b over what the prover writes; squeeze() yields an Fr challenge (the host side of the transcript)
class Transcript {
public:
    void absorb(const void* data, size_t bytes) { h_.update(data, bytes); }
    Fr squeeze() {
        const auto d = h_.digest();
        const uint8_t zero = 0;
        h_.update(&zero, 1);
        return HostFr::from_wide_bytes(d.data());
    }
    // the writer interface ProverSession's shared phases use: m commitments (affine, Montgomery), m public values
    void write_points(const G1* p, size_t m) { absorb(p, m * sizeof(G1)); }
    void common_scalars(const Fr* v, size_t m) { absorb(v, m * sizeof(Fr)); }

private:
    Blake2b h_;
};

// SerdeFormat::Processed encoding of an affine point (Montgomery; the identity (0, 0)): canonical x little-endian and the
// flag bits of include/h2b200.h in byte 31 — the encoding h2b_g1_compress writes and h2b_g1_decompress reads
inline std::array<uint8_t, 32> g1_compress_host(const G1& p) {
    std::array<uint8_t, 32> out{};
    if (HostFq::is_zero(p.x) && HostFq::is_zero(p.y)) {
        out[31] = H2B_G1_FLAG_IDENTITY;
        return out;
    }
    const Fq x = HostFq::to_canonical(p.x), y = HostFq::to_canonical(p.y);
    std::memcpy(out.data(), x.data(), 32);
    if (y[0] & 1) out[31] |= H2B_G1_FLAG_Y_ODD;
    return out;
}

// halo2's Blake2bWrite<_, G1Affine, Challenge255> (transcript.rs, recalled from halo2-axiom 0.5.3): Blake2b-512 personalized
// "Halo2-Transcript"; a point enters as 1 || x || y (canonical little-endian, the identity is an error), a scalar as 2 || its
// canonical bytes, a challenge is 0 absorbed, then the digest of the state as a 512-bit little-endian integer mod r.
// write_point / write_scalar also append the 32-byte encoding (g1_compress_host / canonical) to the proof.
class Blake2bWrite {
public:
    Blake2bWrite() : h_(reinterpret_cast<const uint8_t*>("Halo2-Transcript")) {}
    void common_point(const G1& p) {
        if (HostFq::is_zero(p.x) && HostFq::is_zero(p.y)) throw Error(H2B_ERR_ARG, "Blake2bWrite: the identity cannot enter the transcript");
        const uint8_t prefix = 1;
        const Fq x = HostFq::to_canonical(p.x), y = HostFq::to_canonical(p.y);
        h_.update(&prefix, 1);
        h_.update(x.data(), 32);
        h_.update(y.data(), 32);
    }
    void common_scalar(const Fr& v) {
        const uint8_t prefix = 2;
        const Fr c = HostFr::to_canonical(v);
        h_.update(&prefix, 1);
        h_.update(c.data(), 32);
    }
    void write_point(const G1& p) {
        common_point(p);
        const auto b = g1_compress_host(p);
        out_.insert(out_.end(), b.begin(), b.end());
    }
    void write_scalar(const Fr& v) {
        common_scalar(v);
        const Fr c = HostFr::to_canonical(v);
        const uint8_t* b = reinterpret_cast<const uint8_t*>(c.data());
        out_.insert(out_.end(), b, b + 32);
    }
    Fr squeeze() {
        const uint8_t prefix = 0;
        h_.update(&prefix, 1);
        return HostFr::from_wide_bytes(h_.digest().data());
    }
    void write_points(const G1* p, size_t m) {
        for (size_t i = 0; i < m; i++) write_point(p[i]);
    }
    void common_scalars(const Fr* v, size_t m) {
        for (size_t i = 0; i < m; i++) common_scalar(v[i]);
    }
    // the proof: what transcript.finalize() returns
    const std::vector<uint8_t>& finalize() const { return out_; }

private:
    Blake2b h_;
    std::vector<uint8_t> out_;
};

// ------------------------------------------------------------------------------------------------ device polynomials
class Poly {
public:
    Poly(const Context& ctx, size_t n) : ctx_(&ctx), n_(n) {
        ctx.check(h2b_poly_alloc(ctx.raw(), n, &h_));
        ptr_ = static_cast<char*>(h2b_poly_device_ptr(h_));
    }
    ~Poly() { if (h_) h2b_poly_free(ctx_->raw(), h_); }
    Poly(const Poly&) = delete;
    Poly& operator=(const Poly&) = delete;
    void* at(size_t elem = 0) const { return ptr_ + 32 * elem; }
    size_t len() const { return n_; }
    h2b_poly* raw() const { return h_; }
    void upload(const Fr* host, size_t n, size_t offset = 0) const {
        ctx_->check(h2b_poly_upload(ctx_->raw(), h_, offset, reinterpret_cast<const uint64_t*>(host), n));
    }
    void upload_async(const Fr* pinned, size_t n, size_t offset = 0) const {
        ctx_->check(h2b_poly_upload_async(ctx_->raw(), h_, offset, reinterpret_cast<const uint64_t*>(pinned), n));
    }
    std::vector<Fr> download(size_t offset, size_t n) const {
        std::vector<Fr> out(n);
        if (n) ctx_->check(h2b_poly_download(ctx_->raw(), h_, offset, out[0].data(), n));
        return out;
    }

private:
    const Context* ctx_;
    size_t n_;
    h2b_poly* h_ = nullptr;
    char* ptr_ = nullptr;
};
using PolyPtr = std::unique_ptr<Poly>;

// a column: rows of a device polynomial from `offset` on (an advice column is a slice of the block the assignment kernels write)
struct ColRef {
    const Poly* poly = nullptr;
    size_t offset = 0;
    void* ptr(size_t row = 0) const { return poly->at(offset + row); }
};
// a named device column (tests read them back): where it is and how many rows it has
struct NamedColumn {
    ColRef col;
    size_t rows = 0;
};

// a device buffer of at least m elements, reallocated only when a call needs more than any call before it
inline Poly* grown(const Context& ctx, PolyPtr& p, size_t m) {
    if (!p || p->len() < m) p = std::make_unique<Poly>(ctx, std::max<size_t>(m, 1));
    return p.get();
}
// `bytes` host bytes into p (grown): whole 32-byte elements straight from the caller's array, the last 1..31 bytes through a
// zero-padded element (nothing past the end of the caller's array is read)
inline Poly* upload_bytes(const Context& ctx, PolyPtr& p, const void* host, size_t bytes) {
    if (bytes && !host) throw Error(H2B_ERR_ARG, "upload: null pointer");
    const size_t full = bytes / 32, tail = bytes % 32;
    Poly* d = grown(ctx, p, full + (tail != 0));
    if (full) d->upload(static_cast<const Fr*>(host), full);
    if (tail) {
        Fr last{};
        std::memcpy(last.data(), static_cast<const char*>(host) + 32 * full, tail);
        d->upload(&last, 1, full);
    }
    return d;
}

// ------------------------------------------------------------------------------------------------ the circuit's shape
// What halo2-base's constraint system is for (k, A, L, selector_lookup, I, F): the one place the prover, the check, MockProver
// and keygen read it from.  The selector lookup needs L = 0; blinding factors max(3, queries of a gate column = 4) + 2 = 6.
// Instance columns and constants columns change neither the degree nor the blinding factors, only the number of permutation
// columns (and with it n_sets).  The constants columns enter the permutation first, in the order FlexGateConfig::configure
// enables equality on them, before the gate advice (the range config's lookup advice comes later).
struct CircuitShape {
    CircuitShape(uint32_t k, size_t A, size_t L, bool selector_lookup, size_t I = 0, size_t F = 1)
        : k(k), n(size_t(1) << k), A(A), L(L), I(I), F(F), selector_lookup(selector_lookup && L == 0) {
        degree = L ? 4 : (this->selector_lookup ? 5 : 3);
        chunk = degree - 2;
        ext_k = k + (degree == 3 ? 1 : 2);
        u = n - (bf + 1);
        for (size_t j = 0; j < A; j++) adv_names.push_back("a" + std::to_string(j));
        for (size_t t = 0; t < L; t++) adv_names.push_back("l" + std::to_string(t));
        for (size_t f = 0; f < F; f++) const_names.push_back(f ? "c" + std::to_string(f) : "c");
        perm_cols = const_names;
        perm_cols.insert(perm_cols.end(), adv_names.begin(), adv_names.end());
        for (size_t m = 0; m < I; m++) inst_names.push_back("i" + std::to_string(m));
        perm_cols.insert(perm_cols.end(), inst_names.begin(), inst_names.end());
        n_sets = (perm_cols.size() + chunk - 1) / chunk;
        n_lookups = L ? L : (this->selector_lookup ? 1 : 0);
        for (size_t j = 0; j < A; j++) fixed_names.push_back("q" + std::to_string(j));
        if (this->selector_lookup) fixed_names.push_back("q_lookup");
        if (n_lookups) fixed_names.push_back("table");
        fixed_names.insert(fixed_names.end(), const_names.begin(), const_names.end());
        for (auto& nm : perm_cols) sigma_names.push_back("sigma_" + nm);
    }
    // a permutation column that is a constants column (fixed: it lives in the circuit, not in the session)
    bool is_const(const std::string& nm) const { return std::find(const_names.begin(), const_names.end(), nm) != const_names.end(); }
    uint32_t k, ext_k = 0;
    size_t n, A, L, I, F;
    bool selector_lookup;
    size_t degree = 0, chunk = 0, n_sets = 0, n_lookups = 0, u = 0;
    uint32_t bf = 6;
    // adv: a0.., l0..;  inst: i0..;  const: c, c1..;  perm: const, adv, inst;  fixed: q0.., [q_lookup], [table], const;
    // sigma: sigma_{perm}
    std::vector<std::string> adv_names, inst_names, const_names, perm_cols, fixed_names, sigma_names;
};

// a selector as the gates read it from fixed slot `slot`: the column itself (root 1 of a combination of 1), or, compressed, member
// `root` of a combination of `len`: S prod_{t = 1..len, t != root} (t - S) (halo2's substitution, not normalised; DESIGN §2 (12))
inline ValueSource add_selector(GraphEvaluator& ev, uint32_t slot, size_t root = 1, size_t len = 1) {
    const ValueSource q = ev.add_calculation(Calculation::Store(ValueSource::Fixed(slot, ev.add_rotation(0))));
    ValueSource acc = q;
    for (size_t t = 1; t <= len; t++)
        if (t != root) {
            const Fr c = HostFr::from_canonical(std::array<uint64_t, 4>{t, 0, 0, 0}.data());
            acc = ev.add_calculation(Calculation::Mul(acc, ev.add_calculation(Calculation::Sub(ev.add_constant(c), q))));
        }
    return acc;
}
// calculations of one vertical gate whose selector is a member of a combination of `len` (see ProverCircuit's gate programs)
inline size_t vertical_gate_calculations(size_t len) { return 9 + 2 * (len - 1); }

// the vertical gate q (a0 + a1 a2 - a3) on fixed and advice slot `slot`, advice rotations 0..3 (flex_gate/mod.rs:80-91); q as
// add_selector reads it
inline ValueSource add_vertical_gate(GraphEvaluator& ev, uint32_t slot, size_t root = 1, size_t len = 1) {
    const ValueSource q = add_selector(ev, slot, root, len);
    ValueSource a[4];
    for (int r = 0; r < 4; r++) a[r] = ev.add_calculation(Calculation::Store(ValueSource::Advice(slot, ev.add_rotation(r))));
    const ValueSource sum = ev.add_calculation(Calculation::Add(a[0], ev.add_calculation(Calculation::Mul(a[1], a[2]))));
    return ev.add_calculation(Calculation::Mul(q, ev.add_calculation(Calculation::Sub(sum, a[3]))));
}

// ------------------------------------------------------------------------------------------------ the fixed side of a circuit
class ProverCircuit : public CircuitShape {
public:
    // fixed: Lagrange values (2^k each) by name — q0..q{A-1}, [q_lookup], [table], c, c1..c{F-1}; sigma: one column per
    // permutation column in the order [c, c1.., a0.., l0.., i0..] (F constants columns, I instance columns).
    // compress_selectors: lay the fixed side out as halo2's keygen_vk does (h2b200_selectors.hpp): the selectors q{j} and
    // q_lookup (0/1 values) become the combination columns s0, s1.. and `layout` says where each one went
    ProverCircuit(const Context& ctx, uint32_t k, size_t A, size_t L, bool selector_lookup, const std::map<std::string, std::vector<Fr>>& fixed,
                  const std::vector<std::vector<Fr>>& sigma, size_t I = 0, size_t F = 1, bool compress_selectors = false)
        : ProverCircuit(ctx, k, A, L, selector_lookup, rows_of(fixed, k), rows_of(sigma, k), false, I, F, compress_selectors) {}
    // the same with every column as a pointer to its 2^k rows (nothing is copied on the host)
    ProverCircuit(const Context& ctx, uint32_t k, size_t A, size_t L, bool selector_lookup, const std::map<std::string, const Fr*>& fixed,
                  const std::vector<const Fr*>& sigma, size_t I = 0, size_t F = 1, bool compress_selectors = false)
        : ProverCircuit(ctx, k, A, L, selector_lookup, fixed, sigma, false, I, F, compress_selectors) {}
    // the same with every column as a DEVICE pointer to its 2^k Lagrange values (keygen on the device, h2b200_keygen.hpp): each is
    // copied on the device, then transformed as above
    struct OnDevice {};
    ProverCircuit(OnDevice, const Context& ctx, uint32_t k, size_t A, size_t L, bool selector_lookup,
                  const std::map<std::string, const Fr*>& fixed, const std::vector<const Fr*>& sigma, size_t I = 0, size_t F = 1,
                  bool compress_selectors = false)
        : ProverCircuit(ctx, k, A, L, selector_lookup, fixed, sigma, true, I, F, compress_selectors) {}

private:
    ProverCircuit(const Context& ctx, uint32_t k, size_t A, size_t L, bool selector_lookup, const std::map<std::string, const Fr*>& fixed,
                  const std::vector<const Fr*>& sigma, bool on_device, size_t I, size_t F, bool compress)
        : CircuitShape(k, A, L, selector_lookup, I, F), ctx(ctx) {
        if (sigma.size() != perm_cols.size()) throw Error(H2B_ERR_ARG, "ProverCircuit: one sigma column per permutation column");
        std::vector<Fr> l0(n, Fr{}), ll(n, Fr{}), la(n, Fr{});
        l0[0] = HostFr::one();
        ll[u] = HostFr::one();
        for (size_t i = 0; i < u; i++) la[i] = HostFr::one();
        auto add = [&](const std::string& name, const Fr* arr, bool device) {
            if (!arr) throw Error(H2B_ERR_ARG, "ProverCircuit: column " + name + " is null");
            auto lg = std::make_unique<Poly>(ctx, n), cf = std::make_unique<Poly>(ctx, n), ex = std::make_unique<Poly>(ctx, size_t(1) << ext_k);
            if (device) {
                ctx.check(h2b_poly_copy_dev(ctx.raw(), lg->at(), arr, n));
                ctx.check(h2b_poly_copy_dev(ctx.raw(), cf->at(), arr, n));
            } else {
                lg->upload(arr, n);
                cf->upload(arr, n);
            }
            ctx.check(h2b_lagrange_to_coeff_dev(ctx.raw(), cf->at(), k));
            ctx.check(h2b_coeff_to_extended_dev(ctx.raw(), cf->at(), n, ext_k, ex->at()));
            lagr[name] = std::move(lg);
            coeff[name] = std::move(cf);
            ext[name] = std::move(ex);
        };
        for (auto& nm : fixed_names)
            if (!fixed.count(nm)) throw Error(H2B_ERR_ARG, "ProverCircuit: missing fixed column " + nm);
        std::vector<std::string> selectors;  // selector index order: q0.., q_lookup (convention 14)
        for (size_t j = 0; j < A; j++) selectors.push_back("q" + std::to_string(j));
        if (this->selector_lookup) selectors.push_back("q_lookup");
        std::vector<PolyPtr> staged;  // host selector columns, uploaded for the conflict kernel
        if (!compress) {
            layout = uncompressed_layout(fixed_names, selectors);
            for (auto& nm : fixed_names) add(nm, fixed.at(nm), on_device);
        } else {
            std::vector<const void*> d_sel;
            std::vector<size_t> deg;  // the vertical gate has degree 3; q_lookup is complex (degree 0)
            for (auto& nm : selectors) {
                if (on_device) {
                    d_sel.push_back(fixed.at(nm));
                } else {
                    staged.push_back(std::make_unique<Poly>(ctx, n));
                    staged.back()->upload(fixed.at(nm), n);
                    d_sel.push_back(staged.back()->at());
                }
                deg.push_back(nm == "q_lookup" ? 0 : 3);
            }
            const auto combos = compress_selectors_process(deg, degree, selector_conflicts_dev(ctx, d_sel, k));
            // column order [table], c.. (RangeConfig creates the table before FlexGateConfig its constants columns); query order
            // c.., [table] (enable_equality queries the constants, the lookup queries the table)
            std::vector<std::string> columns, queries = const_names;
            if (n_lookups) {
                columns.push_back("table");
                queries.push_back("table");
            }
            columns.insert(columns.end(), const_names.begin(), const_names.end());
            layout = compressed_layout(columns, queries, selectors, combos);
            for (auto& nm : columns) add(nm, fixed.at(nm), on_device);
            Poly comb(ctx, n);
            for (size_t c = 0; c < combos.size(); c++) {  // S_c = sum_m root_m q_m (the members are active on disjoint rows)
                std::vector<const void*> pp;
                std::vector<Fr> roots;
                for (size_t m = 0; m < combos[c].size(); m++) {
                    pp.push_back(d_sel[combos[c][m]]);
                    roots.push_back(HostFr::from_canonical(std::array<uint64_t, 4>{m + 1, 0, 0, 0}.data()));
                }
                ctx.check(h2b_poly_lincomb_dev(ctx.raw(), pp.data(), roots[0].data(), pp.size(), n, comb.at()));
                add(layout.combinations[c].first, static_cast<const Fr*>(comb.at()), true);
            }
            h2b_ctx_synchronize(ctx.raw());
        }
        for (size_t i = 0; i < perm_cols.size(); i++) add(sigma_names[i], sigma[i], on_device);
        add("l0", l0.data(), false);
        add("l_last", ll.data(), false);
        add("l_active", la.data(), false);
        h2b_ctx_synchronize(ctx.raw());
        // gate programs: GATES_PER_PROGRAM vertical gates each, fewer when compressed selectors add calculations (a program holds
        // at most 64 calculations, one of them the fold); every program continues the Horner fold in y from the previous value,
        // so the chain of programs is the one fold evaluate_h does
        size_t max_len = 1;
        for (auto& e : layout.selectors) max_len = std::max(max_len, e.second.len);
        const size_t per_program = std::min(GATES_PER_PROGRAM, (H2B_GRAPH_MAX_CALCULATIONS - 1) / vertical_gate_calculations(max_len));
        for (size_t j0 = 0; j0 < A; j0 += per_program) {
            GateProgram gp;
            std::vector<ValueSource> parts;
            for (size_t j = j0; j < std::min(A, j0 + per_program); j++) {
                const SelectorAssignment& a = layout.selectors.at("q" + std::to_string(j));
                parts.push_back(add_vertical_gate(gp.ev, uint32_t(j - j0), a.root, a.len));
                gp.cols.push_back(j);
                gp.fixed.push_back(a.column);
            }
            gp.result = gp.ev.add_calculation(Calculation::Horner(ValueSource::PreviousValue(), parts, ValueSource::Y()));
            gate_programs.push_back(std::move(gp));
        }
        // lookup program: (compressed input + beta)(compressed table + gamma); one input / table expression each, so the
        // theta-compression is the expression itself
        if (n_lookups) {
            const uint32_t r0 = lookup_ev.add_rotation(0);
            ValueSource in, tab;
            if (this->selector_lookup) {  // fixed slots [q_lookup, table], advice slot [a0]
                const ValueSource q = lookup_ev.add_calculation(Calculation::Store(ValueSource::Fixed(0, r0)));
                const ValueSource a = lookup_ev.add_calculation(Calculation::Store(ValueSource::Advice(0, r0)));
                in = lookup_ev.add_calculation(Calculation::Mul(q, a));
                tab = lookup_ev.add_calculation(Calculation::Store(ValueSource::Fixed(1, r0)));
            } else {  // fixed slot [table], advice slot [l{t}]
                in = lookup_ev.add_calculation(Calculation::Store(ValueSource::Advice(0, r0)));
                tab = lookup_ev.add_calculation(Calculation::Store(ValueSource::Fixed(0, r0)));
            }
            const ValueSource rg = lookup_ev.add_calculation(Calculation::Add(tab, ValueSource::Gamma()));
            const ValueSource lb = lookup_ev.add_calculation(Calculation::Add(in, ValueSource::Beta()));
            lookup_result = lookup_ev.add_calculation(Calculation::Mul(lb, rg));
        }
    }

public:

    // what ProverSession::check needs beyond a proof, built on the first check: the vertical gate as one program on fixed slot 0 /
    // advice slot 0 (bound to q{j}, a{j} per gate column) and the sigma columns decoded into map[c][r] = c' << k | r' (u32);
    // throws H2B_ERR_ARG naming the first (column, row) whose sigma entry names no cell.  A circuit never checked allocates nothing.
    void prepare_check() const {
        if (check_map) return;
        GraphEvaluator ev;
        const ValueSource res = add_vertical_gate(ev, 0);
        for (auto& e : layout.selectors)  // compressed: one program per (root, len) of a gate's selector
            if (layout.compressed && e.first != "q_lookup" && !check_subst.count({e.second.root, e.second.len})) {
                GraphEvaluator sev;
                const ValueSource sres = add_vertical_gate(sev, 0, e.second.root, e.second.len);
                check_subst[{e.second.root, e.second.len}] = {std::move(sev), sres};
            }
        const size_t npc = perm_cols.size();
        auto map = std::make_unique<Poly>(ctx, (npc * n + 7) / 8);
        Poly rep(ctx, (2 * npc + 3) / 4);  // max_report = 1: count and first row per column
        std::vector<const void*> sig;
        for (auto& nm : sigma_names) sig.push_back(lagr.at(nm)->at());
        permutation_decode_dev(ctx, sig, k, map->at(), 1, rep.at());
        const std::vector<Fr> raw = rep.download(0, rep.len());
        const uint64_t* w = raw[0].data();
        for (size_t c = 0; c < npc; c++)
            if (w[2 * c])
                throw Error(H2B_ERR_ARG, "ProverCircuit: the sigma entry of permutation column " + std::to_string(c) + " (" + perm_cols[c] +
                                             ") at row " + std::to_string(w[2 * c + 1]) + " is not delta^c omega^r for any of the " +
                                             std::to_string(npc) + " permutation columns");
        check_ev = std::move(ev);
        check_result = res;
        check_map = std::move(map);
    }

    // a fixed-side column by name, for tests: "lagr" / "coeff" / "ext" (fixed, sigma and the l0 / l_last / l_active columns)
    // and "sigma_map" (the decoded sigma of the check, built here on first use)
    NamedColumn column(const std::string& table, const std::string& name) const {
        if (table == "sigma_map") {
            prepare_check();
            return {{check_map.get(), 0}, check_map->len()};
        }
        const std::map<std::string, PolyPtr>* t = table == "lagr" ? &lagr : table == "coeff" ? &coeff : table == "ext" ? &ext : nullptr;
        if (!t || !t->count(name)) throw Error(H2B_ERR_ARG, "ProverCircuit: no column " + table + " " + name);
        return {{t->at(name).get(), 0}, t->at(name)->len()};
    }

    // the column that holds selector `sel` (q{j}, q_lookup)
    const std::string& selector_column(const std::string& sel) const { return layout.selectors.at(sel).column; }

    static constexpr size_t GATES_PER_PROGRAM = 5;
    struct GateProgram {
        GraphEvaluator ev;
        ValueSource result{};
        std::vector<size_t> cols;         // the gate columns of the program's advice slots
        std::vector<std::string> fixed;   // the fixed column of each slot (q{j}, or its combination column)
    };
    const Context& ctx;
    SelectorLayout layout;  // where the selectors are, the fixed columns in column and in query order
    std::map<std::string, PolyPtr> lagr, coeff, ext;
    std::vector<GateProgram> gate_programs;
    GraphEvaluator lookup_ev;
    ValueSource lookup_result{};
    mutable GraphEvaluator check_ev;  // prepare_check()
    mutable ValueSource check_result{};
    mutable PolyPtr check_map;
    mutable std::map<std::pair<size_t, size_t>, std::pair<GraphEvaluator, ValueSource>> check_subst;  // compressed: by (root, len)

private:
    static std::map<std::string, const Fr*> rows_of(const std::map<std::string, std::vector<Fr>>& cols, uint32_t k) {
        std::map<std::string, const Fr*> out;
        for (auto& [name, v] : cols) {
            if (v.size() != size_t(1) << k) throw Error(H2B_ERR_ARG, "ProverCircuit: column " + name + " must hold 2^k rows");
            out[name] = v.data();
        }
        return out;
    }
    static std::vector<const Fr*> rows_of(const std::vector<std::vector<Fr>>& cols, uint32_t k) {
        std::vector<const Fr*> out;
        for (auto& v : cols) {
            if (v.size() != size_t(1) << k) throw Error(H2B_ERR_ARG, "ProverCircuit: every sigma column must hold 2^k rows");
            out.push_back(v.data());
        }
        return out;
    }
};

// ------------------------------------------------------------------------------------------------ one proof
// halo2-base's own witness form (one walk over ctx.advice, nothing inverted): the witness holds n for every Rational(n, d)
// cell; rational_index / rational_den are its (virtual-column index, Montgomery d) pairs, indices strictly increasing;
// lookup_index replaces the looked-up values with the virtual-column indices of the cells assign_raw copies, in its order.
struct AssignedWitness {
    std::vector<uint64_t> rational_index;
    std::vector<Fr> rational_den;
    std::vector<uint64_t> lookup_index;
};

// The witness of one proof or check as the caller holds it, pointer + count (nothing is copied on the host): the virtual
// column of the gate cells (Montgomery), break_points as keygen pinned them, and the looked-up cells in assign_raw order (L > 0)
// either as values (lookup_cells) or, in the halo2-base form, as virtual-column indices (lookup_index) — together with the
// (index, d) pairs of its Rational cells (see AssignedWitness).  The public values: instance[m] holds the n_instance[m]
// Montgomery values of instance column m, for the n_instance_columns = I columns of the circuit.
struct WitnessView {
    const Fr* cells = nullptr;
    size_t n_cells = 0;
    const uint64_t* break_points = nullptr;
    size_t n_break_points = 0;
    const Fr* lookup_cells = nullptr;
    const uint64_t* lookup_index = nullptr;
    size_t n_lookup = 0;
    const uint64_t* rational_index = nullptr;
    const Fr* rational_den = nullptr;
    size_t n_rational = 0;
    const Fr* const* instance = nullptr;
    const size_t* n_instance = nullptr;
    size_t n_instance_columns = 0;
    bool assigned_form() const { return n_rational || lookup_index; }
};

// the device side of one witness (ProverSession, MockProver): each buffer is reallocated only when a call needs more than any
// call before it
struct WitnessBuffers {
    PolyPtr cells, rational_index, rational_den, lookups;  // lookups: the looked-up values or their indices
};

// phase 0 up to the advice columns (ProverSession::create_proof and check, MockProver::run): the witness, its Rational pairs and
// its looked-up cells (values or indices) up; with `rational`, the Rational cells become n * d^-1 before anything reads the
// witness; then the assignment into `cols` (the A gate columns, then the L lookup columns, 2^k rows each).  d_verdict[0] /
// d_verdict[1]: the device verdict words of the Rational pairs / of the lookup indices.  random_poly (create_proof): its n
// pinned coefficients go up into `rnd` on the side queue, beside the assignment.  Returns the bytes uploaded.
inline size_t assign_witness(const Context& ctx, const CircuitShape& s, const WitnessView& w, bool rational, uint32_t* d_verdict, void* cols,
                             WitnessBuffers& buf, const Fr* random_poly = nullptr, Poly* rnd = nullptr) {
    h2b_ctx* c = ctx.raw();
    const size_t R = w.n_rational;
    const bool lk_indexed = s.L && w.lookup_index;
    size_t bytes = 32 * w.n_cells;
    upload_bytes(ctx, buf.cells, w.cells, 32 * w.n_cells);
    if (R) {
        upload_bytes(ctx, buf.rational_den, w.rational_den, 32 * R);
        upload_bytes(ctx, buf.rational_index, w.rational_index, 8 * R);
        bytes += 40 * R;
    }
    if (s.L) {
        const size_t each = lk_indexed ? 8 : 32;
        upload_bytes(ctx, buf.lookups, lk_indexed ? static_cast<const void*>(w.lookup_index) : w.lookup_cells, each * w.n_lookup);
        bytes += each * w.n_lookup;
    }
    if (random_poly) {
        ctx.check(h2b_ctx_side_begin(c));
        rnd->upload_async(random_poly, s.n);
        ctx.check(h2b_ctx_side_end(c));
        bytes += 32 * s.n;
    }
    if (rational)  // before anything reads the witness
        ctx.check(h2b_apply_rational_dev(c, buf.cells->at(), w.n_cells, R ? buf.rational_index->at() : nullptr, R ? buf.rational_den->at() : nullptr,
                                         R, d_verdict));
    ctx.check(h2b_assign_columns_dev(c, buf.cells->at(), w.n_cells, w.n_break_points ? w.break_points : nullptr, w.n_break_points, s.k, s.A, cols));
    void* lk_cols = static_cast<char*>(cols) + 32 * s.A * s.n;
    if (lk_indexed)
        ctx.check(h2b_assign_lookups_indexed_dev(c, buf.cells->at(), w.n_cells, buf.lookups->at(), w.n_lookup, s.k, s.L, lk_cols, d_verdict + 1));
    else if (s.L)
        ctx.check(h2b_assign_lookups_dev(c, buf.lookups->at(), w.n_lookup, s.k, s.L, lk_cols));
    return bytes;
}

// the public values of a proof, check or MockProver run (or a builder's instance cells): one column per instance column of the
// shape, each within the usable rows when `bounded` (halo2's InstanceTooLarge)
template <class T>
inline void check_instances(const std::string& who, const CircuitShape& s, const T* const* values, const size_t* counts, size_t n_columns,
                            bool bounded = true) {
    if (n_columns != s.I)
        throw Error(H2B_ERR_ARG, who + ": " + std::to_string(n_columns) + " instance columns for a circuit with " + std::to_string(s.I));
    if (s.I && !(counts && values)) throw Error(H2B_ERR_ARG, who + ": instance columns need their arrays and lengths");
    for (size_t m = 0; m < s.I; m++) {
        if (bounded && counts[m] > s.u)
            throw Error(H2B_ERR_ARG, who + ": InstanceTooLarge: instance column i" + std::to_string(m) + " holds " + std::to_string(counts[m]) +
                                         " values, more than the " + std::to_string(s.u) + " usable rows");
        if (counts[m] && !values[m]) throw Error(H2B_ERR_ARG, who + ": instance column i" + std::to_string(m) + " is null");
    }
}

// (failure count, the first min(count, max_report) failing rows or equality indices, ascending)
using ReportItem = std::pair<uint64_t, std::vector<uint64_t>>;
// n_items reports as the check kernels write them, max_report + 1 words each (the count, then the rows); a failure clears
// `satisfied`
inline std::vector<ReportItem> decode_reports(const uint64_t* w, size_t n_items, size_t max_report, bool& satisfied) {
    std::vector<ReportItem> out;
    for (size_t i = 0; i < n_items; i++) {
        const uint64_t* r = w + (max_report + 1) * i;
        out.push_back({r[0], std::vector<uint64_t>(r + 1, r + 1 + std::min<uint64_t>(r[0], max_report))});
        satisfied = satisfied && r[0] == 0;
    }
    return out;
}

// ProverSession::check: per gate column, lookup and permutation column (perm_cols order) a report
struct CheckReport {
    bool satisfied = true;
    std::vector<ReportItem> gates, lookups, copies;
};

struct Proof {
    std::vector<G1> commitments;
    std::vector<std::pair<std::pair<std::string, int>, Fr>> evals;  // ((column, rotation), value) in query order
    Fr theta{}, beta{}, gamma{}, y{}, x{};
    size_t h2d_bytes = 0, d2h_bytes = 0;
};

class ProverSession {
public:
    // `blind(rows)`: the caller's source of blinding scalars (Montgomery limbs), called in the order the prover blinds its columns
    using BlindSource = std::function<std::vector<Fr>(size_t)>;
    // `allreduce(d_points, m)`: combines the m partial commitments (Jacobian, on the device) of all ranks in place
    using AllReduce = std::function<void(void*, size_t)>;
    // `observer(basis, rows)`: the n rows of every committed polynomial, in commit order (verification runs; synchronises)
    using CommitObserver = std::function<void(int, const std::vector<Fr>&)>;

    ProverSession(const Context& ctx, const ParamsKZG& params, const ProverCircuit& cs) : ctx(ctx), params(params), cs(cs), n_loc(cs.n) {
        const size_t n = cs.n, ne = size_t(1) << cs.ext_k;
        witness_bufs.cells = std::make_unique<Poly>(ctx, n * cs.A);  // steady-state proofs allocate nothing
        if (cs.L) witness_bufs.lookups = std::make_unique<Poly>(ctx, n * cs.L);
        adv_block = std::make_unique<Poly>(ctx, n * (cs.A + cs.L));
        for (size_t j = 0; j < cs.adv_names.size(); j++) lagr[cs.adv_names[j]] = ColRef{adv_block.get(), j * n};
        std::vector<std::string> names = cs.adv_names;
        names.insert(names.end(), cs.inst_names.begin(), cs.inst_names.end());
        for (size_t t = 0; t < cs.n_lookups; t++)
            for (const char* p : {"pa", "ps", "zl"}) names.push_back(p + std::to_string(t));
        for (size_t s = 0; s < cs.n_sets; s++) names.push_back("zp" + std::to_string(s));
        for (auto& nm : names) {
            if (!lagr.count(nm)) lagr[nm] = ColRef{own(n), 0};
            coef[nm] = own(n);
            ext[nm] = own(ne);
        }
        if (cs.selector_lookup) inp = own(n);
        rnd = own(n);
        h = own(ne);
        for (auto& t : tmp) t = own(n);
        for (auto& t : tmp_side) t = own(n);
        d_out = own(49);  // up to 16 commitments; element 48: the verdict words of the halo2-base witness form
        d_status = own(std::max<size_t>(1, cs.n_lookups));
        zero = own(1);  // one zero element (never written)
    }

    // multi-GPU: this rank commits rows [begin, begin + n_loc) of every polynomial (its shard of the SRS) and `allreduce`
    // combines the partial commitments of all ranks after every batched MSM, before they come down; everything else is replicated
    void shard(size_t begin, size_t n_loc, AllReduce allreduce) {
        if (begin + n_loc > cs.n) throw Error(H2B_ERR_ARG, "shard: rows past 2^k");
        shard_begin = begin;
        this->n_loc = n_loc;
        this->allreduce = std::move(allreduce);
    }
    CommitObserver observer;  // empty: proofs download nothing but commitments and evaluations

    // witness: the virtual column of the gate cells (Montgomery), break_points as keygen pinned them, lookup_cells in
    // assign_raw order (L > 0), random_poly: the vanishing argument's random polynomial (n coefficients).
    // form: the halo2-base witness form (see AssignedWitness; then lookup_cells stays empty); a bad index throws once phase 0's
    // commitments are down
    Proof create_proof(const std::vector<Fr>& witness, const std::vector<uint64_t>& break_points, const std::vector<Fr>& lookup_cells,
                       const std::vector<Fr>& random_poly, const BlindSource& blind, const AssignedWitness* form = nullptr) {
        if (random_poly.size() != cs.n) throw Error(H2B_ERR_ARG, "create_proof: the random polynomial must hold 2^k coefficients");
        return create_proof(view(witness, break_points, lookup_cells, form, "create_proof"), random_poly.data(), blind);
    }
    // random_poly: n coefficients in pinned host memory (uploaded asynchronously beside phase 0)
    Proof create_proof(const WitnessView& wit, const Fr* random_poly, const BlindSource& blind) {
        const size_t n = cs.n;
        h2b_ctx* c = ctx.raw();
        Transcript tr;
        Proof res;
        prove_to_x(wit, random_poly, blind, tr, res, "create_proof");
        auto rot = [&](int r) { return rotate(res.x, r); };
        // ---- evaluations at x and its rotations
        const std::vector<Query> queries = this->queries();
        {
            const std::vector<Fr> out = evaluate(queries, res);
            tr.absorb(out.data(), out.size() * sizeof(Fr));
            for (size_t i = 0; i < out.size(); i++) res.evals.push_back({{queries[i].name, queries[i].rot}, out[i]});
        }
        // ---- SHPLONK-shaped opening: per rotation set sum_i v^i p_i, divided by (X - point) for every point of the set
        const Fr v_ch = tr.squeeze(), mu = tr.squeeze();
        std::vector<std::pair<const void*, std::vector<int>>> by_poly;  // first-appearance order
        for (auto& q : queries) {
            auto it = std::find_if(by_poly.begin(), by_poly.end(), [&](auto& e) { return e.first == q.ptr; });
            if (it == by_poly.end()) by_poly.push_back({q.ptr, {q.rot}});
            else it->second.push_back(q.rot);
        }
        std::vector<std::pair<std::vector<int>, std::vector<const void*>>> sets;
        for (auto& e : by_poly) {
            auto it = std::find_if(sets.begin(), sets.end(), [&](auto& s) { return s.first == e.second; });
            if (it == sets.end()) sets.push_back({e.second, {e.first}});
            else it->second.push_back(e.first);
        }
        std::stable_sort(sets.begin(), sets.end(), [](auto& a, auto& b) {
            if (a.first.size() != b.first.size()) return a.first.size() < b.first.size();
            return a.first < b.first;
        });
        auto run_sets = [&](const std::vector<size_t>& which, std::array<Poly*, 3> bufs) {
            Poly *f = bufs[0], *qd = bufs[1], *acc = bufs[2];
            bool first = true;
            for (size_t si : which) {
                auto& [rots, plist] = sets[si];
                std::vector<Fr> sc;
                for (size_t i = 0; i < plist.size(); i++) sc.push_back(HostFr::pow(v_ch, i));
                lincomb(plist, sc, f);
                Poly *src = f, *dst = qd;
                for (int r : rots) {  // successive divisions by (X - point): the quotient by the set's vanishing polynomial
                    const Fr z = rot(r);
                    ctx.check(h2b_kate_division_dev(c, src->at(), n, z.data(), dst->at()));
                    // kate_division writes the n - 1 quotient coefficients; the buffer is reused as an n-coefficient
                    // polynomial (next division, linear combination), so its top coefficient is cleared
                    ctx.check(h2b_poly_copy_dev(c, dst->at(n - 1), zero->at(), 1));
                    std::swap(src, dst);
                }
                const Fr mu_s = HostFr::pow(mu, si);
                if (first) lincomb({src->at()}, {mu_s}, acc);
                else lincomb({acc->at(), src->at()}, {HostFr::one(), mu_s}, acc);
                first = false;
            }
            return !first;
        };
        std::vector<size_t> side_sets, main_sets;  // the rotation sets are independent: every other one on the side queue
        for (size_t i = 0; i < sets.size(); i++) (i % 2 ? main_sets : side_sets).push_back(i);
        ctx.check(h2b_ctx_side_begin(c));
        try {
            run_sets(side_sets, {tmp_side[0], tmp_side[1], tmp_side[2]});
        } catch (...) {
            h2b_ctx_side_end(c);
            throw;
        }
        ctx.check(h2b_ctx_side_end(c));
        const bool have_main = run_sets(main_sets, {tmp[0], tmp[1], tmp[2]});
        ctx.check(h2b_ctx_side_join(c));
        if (have_main) lincomb({tmp[2]->at(), tmp_side[2]->at()}, {HostFr::one(), HostFr::one()}, tmp[2]);
        else ctx.check(h2b_poly_copy_dev(c, tmp[2]->at(), tmp_side[2]->at(), n));
        commit({{H2B_BASIS_MONOMIAL, ColRef{tmp[2], 0}}}, res, &tr);
        const Fr u_ch = tr.squeeze();
        // final quotient: W' = L / (X - u) (the remainder is dropped by kate_division)
        ctx.check(h2b_kate_division_dev(c, tmp[2]->at(), n, u_ch.data(), tmp[3]->at()));
        ctx.check(h2b_poly_copy_dev(c, tmp[3]->at(n - 1), zero->at(), 1));
        commit({{H2B_BASIS_MONOMIAL, ColRef{tmp[3], 0}}}, res, static_cast<Transcript*>(nullptr));
        return res;
    }

    // halo2's create_proof with ProverSHPLONK (halo2-axiom 0.5.3, recalled; DESIGN §2): the same device phases as create_proof
    // up to the h pieces (prove_to_x), written through halo2's Blake2bWrite, then halo2's evaluations and multi-open.
    // vk_repr: the verifying key's transcript_repr, absorbed first (vk.hash_into; the caller computes it from the pinned vk).
    // Returns transcript.finalize(): the bytes gen_proof_with_instances returns.
    std::vector<uint8_t> create_proof_halo2(const WitnessView& wit, const Fr* random_poly, const BlindSource& blind, const Fr& vk_repr) {
        const size_t n = cs.n;
        h2b_ctx* c = ctx.raw();
        Blake2bWrite tr;
        Proof res;
        tr.common_scalar(vk_repr);
        prove_to_x(wit, random_poly, blind, tr, res, "create_proof_halo2");
        // ---- evaluations: advice, fixed, random_poly, sigma, permutation sets, lookups (h(x) is not written)
        for (const Fr& e : evaluate(halo2_evaluations(), res)) tr.write_scalar(e);
        // ---- the vanishing argument opens h(X) = sum_i x^(n i) h_i
        Poly* hx = tmp_side[0];
        {
            std::vector<const void*> pp;
            std::vector<Fr> sc;
            const Fr xn = HostFr::pow(res.x, n);
            Fr s = HostFr::one();
            for (size_t j = 0; j + 1 < cs.degree; j++) {
                pp.push_back(h->at(j * n));
                sc.push_back(s);
                s = HostFr::mul(s, xn);
            }
            lincomb(pp, sc, hx);
        }
        // ---- ProverSHPLONK: commitments grouped by identity in first-appearance order, then by equal point sets
        std::vector<std::pair<const void*, std::vector<int>>> by_poly;
        for (auto& q : halo2_openings(hx)) {
            auto it = std::find_if(by_poly.begin(), by_poly.end(), [&](auto& e) { return e.first == q.ptr; });
            if (it == by_poly.end()) by_poly.push_back({q.ptr, {q.rot}});
            else if (std::find(it->second.begin(), it->second.end(), q.rot) == it->second.end()) it->second.push_back(q.rot);
        }
        std::vector<std::pair<std::vector<int>, std::vector<const void*>>> sets;  // (points as rotations, sorted; polynomials)
        std::vector<int> all;                                                       // T: every point of every set
        for (auto& e : by_poly) {
            const void* ptr = e.first;
            std::vector<int>& rots = e.second;
            std::sort(rots.begin(), rots.end());
            if (rots.size() > H2B_KATE_MULTI_MAX) throw Error(H2B_ERR_ARG, "create_proof_halo2: a rotation set of more than 4 points");
            auto it = std::find_if(sets.begin(), sets.end(), [&](auto& s) { return s.first == rots; });
            if (it == sets.end()) sets.push_back({rots, {ptr}});
            else it->second.push_back(ptr);
            for (int r : rots)
                if (std::find(all.begin(), all.end(), r) == all.end()) all.push_back(r);
        }
        const Fr y = tr.squeeze();
        const Fr v = tr.squeeze();
        auto y_powers = [&](size_t m) {
            std::vector<Fr> p(m, HostFr::one());
            for (size_t i = 1; i < m; i++) p[i] = HostFr::mul(p[i - 1], y);
            return p;
        };
        // h_x = sum_s v^(S-1-s) (q_s - r_s) / Z_{T_s},  q_s = sum_j y^j p_sj  (Horner in v over the sets)
        Poly *f = tmp[0], *qd = tmp[1], *hacc = tmp[2], *lin = tmp[3];
        for (size_t s = 0; s < sets.size(); s++) {
            const auto& [rots, plist] = sets[s];
            lincomb(plist, y_powers(plist.size()), f);
            const size_t m = rots.size();
            std::vector<Fr> pts(m), ws(m, HostFr::one());
            for (size_t j = 0; j < m; j++) pts[j] = rotate(res.x, rots[j]);
            for (size_t j = 0; j < m; j++)
                for (size_t t = 0; t < m; t++)
                    if (t != j) ws[j] = HostFr::mul(ws[j], HostFr::sub(pts[j], pts[t]));
            for (auto& w : ws) w = HostFr::inv(w);
            ctx.check(h2b_kate_division_multi_dev(c, f->at(), n, pts[0].data(), m, ws[0].data(), qd->at()));
            ctx.check(h2b_poly_copy_dev(c, qd->at(n - 1), zero->at(), 1));  // n - 1 coefficients written, used as n
            if (s == 0) ctx.check(h2b_poly_copy_dev(c, hacc->at(), qd->at(), n));
            else lincomb({hacc->at(), qd->at()}, {v, HostFr::one()}, hacc);
        }
        commit({{H2B_BASIS_MONOMIAL, ColRef{hacc, 0}}}, res, &tr);
        const Fr u = tr.squeeze();
        // L = sum_s v^(S-1-s) Z_{T\T_s}(u) q_s - Z_T(u) h_x, without the constants r_s(u): they change only the remainder of
        // L / (X - u), which kate_division drops
        auto vanishing_at_u = [&](const std::vector<int>& rots) {
            Fr z = HostFr::one();
            for (int r : rots) z = HostFr::mul(z, HostFr::sub(u, rotate(res.x, r)));
            return z;
        };
        std::vector<const void*> lp;
        std::vector<Fr> ls;
        Fr vs = HostFr::one();  // v^(S-1-s), s from the last set down
        for (size_t s = sets.size(); s-- > 0;) {
            const auto& [rots, plist] = sets[s];
            std::vector<int> diff;
            for (int r : all)
                if (std::find(rots.begin(), rots.end(), r) == rots.end()) diff.push_back(r);
            const Fr coef = HostFr::mul(vs, vanishing_at_u(diff));
            const std::vector<Fr> yp = y_powers(plist.size());
            for (size_t j = 0; j < plist.size(); j++) {
                lp.push_back(plist[j]);
                ls.push_back(HostFr::mul(coef, yp[j]));
            }
            vs = HostFr::mul(vs, v);
        }
        lp.push_back(hacc->at());
        ls.push_back(HostFr::neg(vanishing_at_u(all)));
        lincomb(lp, ls, lin);
        // W' = L / (X - u)
        ctx.check(h2b_kate_division_dev(c, lin->at(), n, u.data(), f->at()));
        ctx.check(h2b_poly_copy_dev(c, f->at(n - 1), zero->at(), 1));
        commit({{H2B_BASIS_MONOMIAL, ColRef{f, 0}}}, res, &tr);
        return tr.finalize();
    }

    // commitments per proof, in commit order: advice | permuted pairs | product columns + random | h pieces | two openings
    size_t commitments_per_proof() const {
        return cs.adv_names.size() + 2 * cs.n_lookups + (cs.n_sets + cs.n_lookups + 1) + (cs.degree - 1) + 2;
    }
    // the evaluations of a proof, in the order they enter the transcript: (column, rotation) and the coefficients evaluated
    struct Query {
        std::string name;
        const void* ptr;
        int rot;
    };
    std::vector<Query> queries() const {
        const int last = -int(cs.bf + 1);
        std::vector<Query> q;
        auto add = [&](const std::string& nm, int r) { q.push_back({nm, coef.at(nm)->at(), r}); };
        for (size_t j = 0; j < cs.A; j++)
            for (int r : {0, 1, 2, 3}) add("a" + std::to_string(j), r);
        for (size_t t = 0; t < cs.L; t++) add("l" + std::to_string(t), 0);
        for (auto& nm : cs.layout.fixed_queries) q.push_back({nm, cs.coeff.at(nm)->at(), 0});
        for (auto& nm : cs.sigma_names) q.push_back({nm, cs.coeff.at(nm)->at(), 0});
        for (size_t s = 0; s < cs.n_sets; s++) {  // every set at x and omega x; all but the last one also at omega^last x
            const std::string nm = "zp" + std::to_string(s);
            add(nm, 0);
            add(nm, 1);
            if (s + 1 < cs.n_sets) add(nm, last);
        }
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const std::string ts = std::to_string(t);
            add("pa" + ts, 0);
            add("pa" + ts, -1);
            add("ps" + ts, 0);
            add("zl" + ts, 0);
            add("zl" + ts, 1);
        }
        for (size_t j = 0; j + 1 < cs.degree; j++) q.push_back({"h" + std::to_string(j), h->at(j * cs.n), 0});
        q.push_back({"rnd", rnd->at(), 0});
        return q;
    }

    // the evaluations of create_proof_halo2 in the order halo2 writes them: advice (advice_queries), fixed (fixed_queries),
    // random_poly, sigma, per permutation set z(x), z(omega x) and, but for the last set, z(omega^last x), per lookup z(x),
    // z(omega x), A'(x), A'(omega^-1 x), S'(x)
    std::vector<Query> halo2_evaluations() const {
        const int last = -int(cs.bf + 1);
        std::vector<Query> q = advice_queries();
        for (auto& nm : cs.layout.fixed_queries) q.push_back({nm, cs.coeff.at(nm)->at(), 0});
        q.push_back({"rnd", rnd->at(), 0});
        for (auto& nm : cs.sigma_names) q.push_back({nm, cs.coeff.at(nm)->at(), 0});
        for (size_t s = 0; s < cs.n_sets; s++) {
            const std::string nm = "zp" + std::to_string(s);
            for (int r : {0, 1}) q.push_back({nm, coef.at(nm)->at(), r});
            if (s + 1 < cs.n_sets) q.push_back({nm, coef.at(nm)->at(), last});
        }
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const std::string ts = std::to_string(t);
            for (auto [nm, r] : std::initializer_list<std::pair<const char*, int>>{{"zl", 0}, {"zl", 1}, {"pa", 0}, {"pa", -1}, {"ps", 0}})
                q.push_back({nm + ts, coef.at(nm + ts)->at(), r});
        }
        return q;
    }
    // the opening queries of create_proof_halo2 in halo2's order (it fixes the rotation sets): advice, permutation sets at x
    // and omega x then omega^last x for the sets in reverse order but the last, per lookup z(x), A'(x), S'(x), A'(omega^-1 x),
    // z(omega x), fixed, sigma, h(X) = `hx`, random_poly
    std::vector<Query> halo2_openings(const Poly* hx) const {
        const int last = -int(cs.bf + 1);
        std::vector<Query> q = advice_queries();
        for (size_t s = 0; s < cs.n_sets; s++) {
            const std::string nm = "zp" + std::to_string(s);
            for (int r : {0, 1}) q.push_back({nm, coef.at(nm)->at(), r});
        }
        for (size_t s = cs.n_sets; s-- > 1;) {
            const std::string nm = "zp" + std::to_string(s - 1);
            q.push_back({nm, coef.at(nm)->at(), last});
        }
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const std::string ts = std::to_string(t);
            for (auto [nm, r] : std::initializer_list<std::pair<const char*, int>>{{"zl", 0}, {"pa", 0}, {"ps", 0}, {"pa", -1}, {"zl", 1}})
                q.push_back({nm + ts, coef.at(nm + ts)->at(), r});
        }
        for (auto& nm : cs.layout.fixed_queries) q.push_back({nm, cs.coeff.at(nm)->at(), 0});
        for (auto& nm : cs.sigma_names) q.push_back({nm, cs.coeff.at(nm)->at(), 0});
        q.push_back({"h", hx->at(), 0});
        q.push_back({"rnd", rnd->at(), 0});
        return q;
    }
    std::vector<Query> advice_queries() const {
        std::vector<Query> q;
        for (size_t j = 0; j < cs.A; j++)
            for (int r : {0, 1, 2, 3}) q.push_back({"a" + std::to_string(j), coef.at("a" + std::to_string(j))->at(), r});
        for (size_t t = 0; t < cs.L; t++) q.push_back({"l" + std::to_string(t), coef.at("l" + std::to_string(t))->at(), 0});
        return q;
    }

    // MockProver::verify for this circuit: the witness as for create_proof, the same assignment, no blinding, no random
    // polynomial, no transcript; rows >= u read as 0.  Every report comes down in one copy; a bad index of the halo2-base form
    // throws H2B_ERR_ARG.
    CheckReport check(const std::vector<Fr>& witness, const std::vector<uint64_t>& break_points, const std::vector<Fr>& lookup_cells,
                      const AssignedWitness* form = nullptr, size_t max_report = 16) {
        return check(view(witness, break_points, lookup_cells, form, "check"), max_report);
    }
    CheckReport check(const WitnessView& wit, size_t max_report = 16) {
        const uint32_t k = cs.k;
        const size_t n = cs.n, u = cs.u, A = cs.A, L = cs.L;
        h2b_ctx* c = ctx.raw();
        check_inputs(wit, "check", cs);
        if (max_report < 1 || max_report > H2B_CHECK_MAX_REPORT) throw Error(H2B_ERR_ARG, "check: max_report out of range");
        cs.prepare_check();
        assign_witness(ctx, cs, wit, wit.assigned_form(), verdict_words(), adv_block->at(), witness_bufs);
        upload_instances(wit);
        Poly* zero_rows = grown(ctx, check_zero, n - u);  // zero-filled, never written
        for (auto& nm : cs.adv_names) ctx.check(h2b_poly_copy_dev(c, lagr[nm].ptr(u), zero_rows->at(), n - u));
        // report block: element 0 = the witness-form verdict words, then max_report + 1 words per gate, lookup, permutation column
        const size_t W = max_report + 1, npc = cs.perm_cols.size(), n_items = A + cs.n_lookups + npc, elems = 1 + (n_items * W + 3) / 4;
        Poly* rep = grown(ctx, check_rep, elems);
        auto at = [&](size_t i) { return static_cast<char*>(rep->at(1)) + 8 * W * i; };
        if (wit.assigned_form()) ctx.check(h2b_poly_copy_dev(c, rep->at(), verdict_words(), 1));
        for (size_t j = 0; j < A; j++) {
            const SelectorAssignment& sa = cs.layout.selectors.at("q" + std::to_string(j));
            const GraphEvaluator& gev = cs.layout.compressed ? cs.check_subst.at({sa.root, sa.len}).first : cs.check_ev;
            const ValueSource gres = cs.layout.compressed ? cs.check_subst.at({sa.root, sa.len}).second : cs.check_result;
            const BoundGraph g(gev, gres, {cs.lagr.at(sa.column)->at()}, {lagr["a" + std::to_string(j)].ptr()});
            check_graph_dev(ctx, *g.get(), k, u, max_report, at(j));
        }
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const void* in = lagr[L ? "l" + std::to_string(t) : "a0"].ptr();
            if (L == 0) {
                ctx.check(h2b_fr_mul_elementwise_dev(c, cs.lagr.at(cs.selector_column("q_lookup"))->at(), in, n, inp->at()));
                in = inp->at();
            }
            check_lookup_dev(ctx, in, cs.lagr.at("table")->at(), k, u, max_report, at(A + t));
        }
        std::vector<const void*> cols;
        for (auto& nm : cs.const_names) cols.push_back(cs.lagr.at(nm)->at());
        for (auto& nm : cs.adv_names) cols.push_back(lagr[nm].ptr());
        for (auto& nm : cs.inst_names) cols.push_back(lagr[nm].ptr());
        check_copies_dev(ctx, cols, cs.check_map->at(), k, max_report, at(A + cs.n_lookups));
        const std::vector<Fr> raw = rep->download(0, elems);
        const uint64_t* w = raw[0].data();
        if (wit.assigned_form()) {
            const uint32_t rat_bad = uint32_t(w[0]), lk_bad = L && wit.lookup_index ? uint32_t(w[0] >> 32) : 0;
            if (rat_bad || lk_bad) witness_error(rat_bad, lk_bad, "check");
        }
        CheckReport out;
        const std::vector<ReportItem> items = decode_reports(w + 4, n_items, max_report, out.satisfied);
        out.gates.assign(items.begin(), items.begin() + A);
        out.lookups.assign(items.begin() + A, items.begin() + A + cs.n_lookups);
        out.copies.assign(items.begin() + A + cs.n_lookups, items.end());
        return out;
    }

    // a session column by name, for tests: "lagr" / "coef" / "ext" by column name, "h" (the quotient: values on the extended
    // coset, then the coefficients of its pieces) and "check_report" (the report block of the last check)
    NamedColumn column(const std::string& table, const std::string& name) const {
        if (table == "lagr" && lagr.count(name)) return {lagr.at(name), cs.n};
        if (table == "coef" && coef.count(name)) return {{coef.at(name), 0}, cs.n};
        if (table == "ext" && ext.count(name)) return {{ext.at(name), 0}, ext.at(name)->len()};
        if (table == "h") return {{h, 0}, h->len()};
        if (table == "check_report" && check_rep) return {{check_rep.get(), 0}, check_rep->len()};
        throw Error(H2B_ERR_ARG, "ProverSession: no column " + table + " " + name);
    }

private:
    // phase 0 up to the commitments of the h pieces and the challenge x, the device work create_proof and create_proof_halo2
    // share: `tr` (Transcript or Blake2bWrite) takes the public values (common_scalars) and every commitment (write_points);
    // res receives the commitments, the challenges theta .. x and the byte counts
    template <class TR>
    void prove_to_x(const WitnessView& wit, const Fr* random_poly, const BlindSource& blind, TR& tr, Proof& res, const std::string& who) {
        const uint32_t k = cs.k, ext_k = cs.ext_k, bf = cs.bf;
        const size_t n = cs.n, u = cs.u, L = cs.L;
        h2b_ctx* c = ctx.raw();
        check_inputs(wit, who, cs);
        if (!random_poly) throw Error(H2B_ERR_ARG, who + ": null random polynomial");
        uint64_t verdict = 0;  // phase 0: the verdict words, read with the first download of its commitments
        auto blind_col = [&](const ColRef& col, size_t first_row) {
            const std::vector<Fr> b = blind(n - first_row);
            if (b.size() != n - first_row) throw Error(H2B_ERR_ARG, "blind source returned the wrong number of rows");
            ctx.check(h2b_poly_upload(c, col.poly->raw(), col.offset + first_row, b[0].data(), b.size()));
            res.h2d_bytes += b.size() * 32;
        };
        auto side_transforms = [&](const std::vector<std::string>& names) {
            ctx.check(h2b_ctx_side_begin(c));
            try {
                for (auto& nm : names) {
                    ctx.check(h2b_poly_copy_dev(c, coef[nm]->at(), lagr[nm].ptr(), n));
                    ctx.check(h2b_lagrange_to_coeff_dev(c, coef[nm]->at(), k));
                    ctx.check(h2b_coeff_to_extended_dev(c, coef[nm]->at(), n, ext_k, ext[nm]->at()));
                }
            } catch (...) {
                h2b_ctx_side_end(c);
                throw;
            }
            ctx.check(h2b_ctx_side_end(c));
        };

        // ---- phase 0: the public values into the transcript; witness up, assignment, advice commitments (the random polynomial
        // and the instance columns go up beside them)
        for (size_t m = 0; m < cs.I; m++) tr.common_scalars(wit.instance[m], wit.n_instance[m]);
        res.h2d_bytes += assign_witness(ctx, cs, wit, wit.assigned_form(), verdict_words(), adv_block->at(), witness_bufs, random_poly, rnd);
        res.h2d_bytes += upload_instances(wit);
        std::vector<std::pair<int, ColRef>> items;
        for (auto& nm : cs.adv_names) {
            blind_col(lagr[nm], u);
            items.push_back({H2B_BASIS_LAGRANGE, lagr[nm]});
        }
        commit(items, res, &tr, wit.assigned_form() ? &verdict : nullptr);
        const uint32_t rat_bad = uint32_t(verdict), lk_bad = L && wit.lookup_index ? uint32_t(verdict >> 32) : 0;
        if (rat_bad || lk_bad) {
            h2b_ctx_side_join(c);  // nothing of this proof stays in flight behind the error
            h2b_ctx_synchronize(c);
            witness_error(rat_bad, lk_bad, who);
        }
        res.theta = tr.squeeze();
        ctx.check(h2b_ctx_side_join(c));  // the random polynomial arrived while phase 0 ran
        std::vector<std::string> phase0 = cs.adv_names;
        phase0.insert(phase0.end(), cs.inst_names.begin(), cs.inst_names.end());
        side_transforms(phase0);
        // ---- lookups: compressed input, permuted pair (enqueue only; the verdict words are read after this phase's commitments)
        std::vector<void*> lk_in;
        items.clear();
        std::vector<std::string> perm_names;
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const std::string ts = std::to_string(t);
            if (L == 0) {
                ctx.check(h2b_fr_mul_elementwise_dev(c, cs.lagr.at(cs.selector_column("q_lookup"))->at(), lagr["a0"].ptr(), n, inp->at()));
                lk_in.push_back(inp->at());
            } else {
                lk_in.push_back(lagr["l" + ts].ptr());
            }
            const ColRef &pa = lagr["pa" + ts], &ps = lagr["ps" + ts];
            ctx.check(h2b_permute_expression_pair_async_dev(c, lk_in[t], cs.lagr.at("table")->at(), k, bf, pa.ptr(), ps.ptr(),
                                                            static_cast<uint32_t*>(d_status->at(t))));
            blind_col(pa, u);
            blind_col(ps, u);
            items.push_back({H2B_BASIS_LAGRANGE, pa});
            items.push_back({H2B_BASIS_LAGRANGE, ps});
            perm_names.push_back("pa" + ts);
            perm_names.push_back("ps" + ts);
        }
        if (cs.n_lookups) {
            commit(items, res, &tr);
            for (auto& w : d_status->download(0, cs.n_lookups))
                if (w[0]) throw Error(H2B_ERR_UNSATISFIED, "permute_expression_pair: an input value is not in the table (ConstraintSystemFailure)");
            res.d2h_bytes += 32 * cs.n_lookups;
        }
        res.beta = tr.squeeze();
        res.gamma = tr.squeeze();
        side_transforms(perm_names);
        // ---- product columns + the vanishing argument's random polynomial
        auto col_lagr = [&](const std::string& nm) -> void* { return cs.is_const(nm) ? cs.lagr.at(nm)->at() : lagr[nm].ptr(); };
        for (size_t s = 0; s < cs.n_sets; s++) {
            std::vector<const void*> cols, sig;
            for (size_t i = s * cs.chunk; i < std::min(cs.perm_cols.size(), (s + 1) * cs.chunk); i++) {
                cols.push_back(col_lagr(cs.perm_cols[i]));
                sig.push_back(cs.lagr.at("sigma_" + cs.perm_cols[i])->at());
            }
            const void* start = s == 0 ? nullptr : lagr["zp" + std::to_string(s - 1)].ptr(u);  // chained through the previous set's closing value
            ctx.check(h2b_permutation_product_dev(c, cols.data(), sig.data(), cols.size(), s * cs.chunk, res.beta.data(), res.gamma.data(), k, bf, start,
                                                  lagr["zp" + std::to_string(s)].ptr()));
        }
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const std::string ts = std::to_string(t);
            ctx.check(h2b_lookup_product_dev(c, lk_in[t], cs.lagr.at("table")->at(), lagr["pa" + ts].ptr(), lagr["ps" + ts].ptr(), res.beta.data(),
                                             res.gamma.data(), k, bf, lagr["zl" + ts].ptr()));
        }
        std::vector<std::string> prod_names;
        for (size_t s = 0; s < cs.n_sets; s++) prod_names.push_back("zp" + std::to_string(s));
        for (size_t t = 0; t < cs.n_lookups; t++) prod_names.push_back("zl" + std::to_string(t));
        items.clear();
        for (auto& nm : prod_names) {
            blind_col(lagr[nm], u + 1);
            items.push_back({H2B_BASIS_LAGRANGE, lagr[nm]});
        }
        side_transforms(prod_names);  // beside the commitments below
        items.push_back({H2B_BASIS_MONOMIAL, ColRef{rnd, 0}});
        commit(items, res, &tr);
        res.y = tr.squeeze();
        ctx.check(h2b_ctx_side_join(c));  // every column is now in coefficient and extended form
        // ---- quotient: gate, permutation and lookup terms folded with y on the extended coset
        Challenges ch;
        ch.beta = res.beta; ch.gamma = res.gamma; ch.theta = res.theta; ch.y = res.y;
        ctx.check(h2b_poly_zero(c, h->raw()));
        for (auto& gp : cs.gate_programs) {
            std::vector<const void*> fx, ad;
            for (size_t i = 0; i < gp.cols.size(); i++) {
                fx.push_back(cs.ext.at(gp.fixed[i])->at());
                ad.push_back(ext["a" + std::to_string(gp.cols[i])]->at());
            }
            const BoundGraph g(gp.ev, gp.result, fx, ad, ch);
            ctx.check(h2b_quotient_graph_dev(c, g.get(), k, ext_k, h->at()));
        }
        {
            std::vector<const void*> tz, tc, ts;
            for (size_t s = 0; s < cs.n_sets; s++) tz.push_back(ext["zp" + std::to_string(s)]->at());
            for (auto& nm : cs.perm_cols) {
                tc.push_back(cs.is_const(nm) ? cs.ext.at(nm)->at() : ext[nm]->at());
                ts.push_back(cs.ext.at("sigma_" + nm)->at());
            }
            ctx.check(h2b_permutation_fold_dev(c, tz.data(), cs.n_sets, tc.data(), ts.data(), tc.size(), cs.chunk, cs.ext.at("l0")->at(),
                                               cs.ext.at("l_last")->at(), cs.ext.at("l_active")->at(), res.beta.data(), res.gamma.data(), res.y.data(), bf, k,
                                               ext_k, h->at()));
        }
        for (size_t t = 0; t < cs.n_lookups; t++) {
            const std::string ts = std::to_string(t);
            std::vector<const void*> fx, ad;
            if (L == 0) {
                fx = {cs.ext.at(cs.selector_column("q_lookup"))->at(), cs.ext.at("table")->at()};
                ad = {ext["a0"]->at()};
            } else {
                fx = {cs.ext.at("table")->at()};
                ad = {ext["l" + ts]->at()};
            }
            const BoundGraph g(cs.lookup_ev, cs.lookup_result, fx, ad, ch);
            ctx.check(h2b_lookup_fold_dev(c, g.get(), ext["zl" + ts]->at(), ext["pa" + ts]->at(), ext["ps" + ts]->at(), cs.ext.at("l0")->at(),
                                          cs.ext.at("l_last")->at(), cs.ext.at("l_active")->at(), k, ext_k, h->at()));
        }
        ctx.check(h2b_divide_by_vanishing_poly_dev(c, h->at(), k, ext_k));
        ctx.check(h2b_extended_to_coeff_dev(c, h->at(), ext_k));
        const size_t pieces = cs.degree - 1;
        items.clear();
        for (size_t j = 0; j < pieces; j++) items.push_back({H2B_BASIS_MONOMIAL, ColRef{h, j * n}});
        commit(items, res, &tr);
        res.x = tr.squeeze();
    }
    // commits `items` (batched MSMs of at most 16), appends the affine points to res.commitments and writes them to `tr` (none:
    // null); with `verdict`, the first download also brings the phase-0 verdict words
    template <class TR>
    void commit(const std::vector<std::pair<int, ColRef>>& items, Proof& res, TR* tr, uint64_t* verdict = nullptr) {
        h2b_ctx* c = ctx.raw();
        for (size_t lo = 0; lo < items.size(); lo += 16) {
            const size_t m = std::min<size_t>(16, items.size() - lo);
            std::vector<const void*> ptrs(m);
            std::vector<int> bs(m);
            for (size_t i = 0; i < m; i++) { bs[i] = items[lo + i].first; ptrs[i] = items[lo + i].second.ptr(shard_begin); }
            ctx.check(h2b_msm_g1_batch_dev(c, params.raw(), bs.data(), ptrs.data(), m, n_loc, d_out->at()));
            if (allreduce) allreduce(d_out->at(), m);
            if (observer) {
                ctx.check(h2b_ctx_synchronize(c));
                for (size_t i = 0; i < m; i++) observer(bs[i], items[lo + i].second.poly->download(items[lo + i].second.offset, cs.n));
            }
            const size_t cnt = verdict && lo == 0 ? 49 : m * 3;
            std::vector<G1> out(m);
            if (cnt == 49) {
                std::vector<Fr> raw = d_out->download(0, 49);
                std::memcpy(out[0].x.data(), raw.data(), m * sizeof(G1));
                *verdict = raw[48][0];
            } else {
                ctx.check(h2b_poly_download(c, d_out->raw(), 0, out[0].x.data(), m * 3));
            }
            res.d2h_bytes += cnt * 32;
            g1_normalize_host_batch(out.data(), m);  // affine form: what the transcript and the proof hold
            if (tr) tr->write_points(out.data(), m);
            res.commitments.insert(res.commitments.end(), out.begin(), out.end());
        }
    }
    // out = sum_i scalars[i] ptrs[i] over n coefficients (h2b_poly_lincomb takes at most 32 polynomials a call)
    void lincomb(const std::vector<const void*>& ptrs, const std::vector<Fr>& scalars, Poly* out) {
        bool first = true;
        for (size_t lo = 0; lo < ptrs.size(); lo += 31) {
            std::vector<const void*> pp(ptrs.begin() + lo, ptrs.begin() + std::min(ptrs.size(), lo + 31));
            std::vector<Fr> sc(scalars.begin() + lo, scalars.begin() + std::min(ptrs.size(), lo + 31));
            if (!first) { pp.insert(pp.begin(), out->at()); sc.insert(sc.begin(), HostFr::one()); }
            ctx.check(h2b_poly_lincomb_dev(ctx.raw(), pp.data(), sc[0].data(), pp.size(), cs.n, out->at()));
            first = false;
        }
    }
    // x omega^r
    Fr rotate(const Fr& x, int r) const {
        const long long n = (long long)cs.n;
        return HostFr::mul(x, HostFr::pow(HostFr::omega(cs.k), uint64_t(((r % n) + n) % n)));
    }
    // the queries' values at x omega^rot, in one batch
    std::vector<Fr> evaluate(const std::vector<Query>& q, Proof& res) {
        const size_t m = q.size();
        std::vector<const void*> polys(m);
        std::vector<Fr> xs(m), out(m);
        for (size_t i = 0; i < m; i++) { polys[i] = q[i].ptr; xs[i] = rotate(res.x, q[i].rot); }
        ctx.check(h2b_eval_polynomial_batch_dev(ctx.raw(), polys.data(), xs[0].data(), m, cs.n, out[0].data()));
        res.d2h_bytes += m * 32;
        return out;
    }
    static WitnessView view(const std::vector<Fr>& witness, const std::vector<uint64_t>& break_points, const std::vector<Fr>& lookup_cells,
                            const AssignedWitness* form, const std::string& who) {
        WitnessView w;
        w.cells = witness.data();
        w.n_cells = witness.size();
        w.break_points = break_points.empty() ? nullptr : break_points.data();
        w.n_break_points = break_points.size();
        w.lookup_cells = lookup_cells.data();
        w.n_lookup = lookup_cells.size();
        if (form) {
            if (form->rational_index.size() != form->rational_den.size())
                throw Error(H2B_ERR_ARG, who + ": rational_index and rational_den differ in length");
            w.rational_index = form->rational_index.data();
            w.rational_den = form->rational_den.data();
            w.n_rational = form->rational_index.size();
            if (!form->lookup_index.empty()) {
                if (!lookup_cells.empty()) throw Error(H2B_ERR_ARG, who + ": pass the looked-up cells either as values or as indices");
                w.lookup_cells = nullptr;
                w.lookup_index = form->lookup_index.data();
                w.n_lookup = form->lookup_index.size();
            }
        }
        return w;
    }
    static void check_inputs(const WitnessView& w, const std::string& who, const CircuitShape& s) {
        if (w.lookup_cells && w.lookup_index) throw Error(H2B_ERR_ARG, who + ": pass the looked-up cells either as values or as indices");
        if (w.n_rational && !(w.rational_index && w.rational_den))
            throw Error(H2B_ERR_ARG, who + ": n_rational > 0 needs rational_index and rational_den");
        check_instances(who, s, w.instance, w.n_instance, w.n_instance_columns);
    }
    // instance column m: rows [0, n_instance[m]) = its public values, the rest zero (beside phase 0 on the main queue)
    size_t upload_instances(const WitnessView& w) {
        size_t bytes = 0;
        for (size_t m = 0; m < cs.I; m++) {
            const ColRef& col = lagr[cs.inst_names[m]];
            ctx.check(h2b_poly_zero(ctx.raw(), col.poly->raw()));
            if (w.n_instance[m]) col.poly->upload(w.instance[m], w.n_instance[m]);
            bytes += 32 * w.n_instance[m];
        }
        return bytes;
    }
    [[noreturn]] static void witness_error(uint32_t rat_bad, uint32_t lk_bad, const std::string& who) {
        std::string why;
        if (rat_bad & 1) why += "; a Rational index is >= the witness length";
        if (rat_bad & 2) why += "; the Rational indices do not strictly increase";
        if (lk_bad & 1) why += "; a lookup index is >= the witness length";
        throw Error(H2B_ERR_ARG, who + why);
    }
    // phase 0 of the halo2-base witness form: the verdict words, read with the first download of its commitments
    uint32_t* verdict_words() const { return static_cast<uint32_t*>(d_out->at(48)); }
    Poly* own(size_t m) {
        owned.push_back(std::make_unique<Poly>(ctx, m));
        return owned.back().get();
    }

    const Context& ctx;
    const ParamsKZG& params;
    const ProverCircuit& cs;
    size_t shard_begin = 0, n_loc;  // shard()
    AllReduce allreduce;
    std::vector<PolyPtr> owned;
    WitnessBuffers witness_bufs;
    PolyPtr adv_block;
    PolyPtr check_zero, check_rep;     // check(): zero rows, the report block
    std::map<std::string, ColRef> lagr;
    std::map<std::string, Poly*> coef, ext;
    Poly *inp = nullptr, *rnd = nullptr, *h = nullptr, *d_out = nullptr, *d_status = nullptr, *zero = nullptr;
    std::array<Poly*, 4> tmp{};
    std::array<Poly*, 3> tmp_side{};
};

}  // namespace h2b
