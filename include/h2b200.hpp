// h2b200.hpp — C++ host-side mirror of the prover interfaces halo2-lib reaches through `halo2_base::halo2_proofs`
// (halo2-base/src/lib.rs:25-28) for the create_proof hot path, implemented on top of the C ABI in h2b200.h.
//
// The reference's host code is Rust (halo2-axiom 0.5.3 / halo2curves-axiom 0.7.3, not vendored; no Rust toolchain in
// this image), so this header restates the same operator surface in C++ with the same names, argument meaning
// and failure behaviour; the Rust binding a maintainer would add is shown in INTEGRATION.md.
//
//   halo2curves::msm::best_multiexp(coeffs, bases) -> G1            h2b::best_multiexp
//   halo2_proofs::arithmetic::best_fft(a, omega, log_n)             h2b::best_fft
//   halo2_proofs::poly::kzg::commitment::ParamsKZG::{commit, commit_lagrange}      h2b::ParamsKZG
//   halo2_proofs::poly::EvaluationDomain::{new, lagrange_to_coeff, coeff_to_lagrange, coeff_to_extended,
//                                           extended_to_coeff}                      h2b::EvaluationDomain
//   halo2_base::gates::flex_gate::threads::single_phase::assign_witnesses           h2b::assign_witnesses
//       (halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312)
//   halo2_base::virtual_region::lookups::LookupAnyManager::assign_raw               h2b::assign_lookups
//       (halo2-base/src/virtual_region/lookups.rs:130-155)
//
//   ff::BatchInvert::batch_invert, the grand-product column of the permutation / lookup provers   h2b::batch_invert, grand_product
//   halo2_proofs::plonk::lookup::prover::permute_expression_pair                      h2b::permute_expression_pair
//   halo2_proofs::plonk::evaluation::{GraphEvaluator, Evaluator::evaluate_h}          h2b::GraphEvaluator, quotient_graph,
//                                                                                     permutation_fold, lookup_fold
//   halo2_proofs::poly::EvaluationDomain::divide_by_vanishing_poly                    h2b::divide_by_vanishing_poly
//   halo2_proofs::arithmetic::{eval_polynomial, kate_division}                        h2b::eval_polynomial, kate_division
//   halo2_proofs::poly::kzg::commitment::g_to_lagrange                                h2b::g_to_lagrange
//   ParamsKZG::{setup (ChaCha20Rng seeded), write, read}, Params::downsize              h2b::ParamsKZG::{setup_seeded, write,
//                                                                                     read, read_downsized, downsize}
//   halo2_base::utils::fs::gen_srs (read_or_create_srs, utils/mod.rs:413-443)         h2b::gen_srs
//
// Where the Rust code panics (`expect("prover should not fail")`, halo2-base/src/utils/testing.rs:48; index out of
// bounds in assign_witnesses) these wrappers throw h2b::Error; nothing is computed on the CPU.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "h2b200.h"

namespace h2b {

using Fr = std::array<uint64_t, 4>;        // [u64;4] LE Montgomery (halo2-base/src/utils/mod.rs:332-377)
using Fq = std::array<uint64_t, 4>;
struct G1Affine { Fq x, y; };              // identity = (0,0)
struct G1 { Fq x, y, z; };                 // Jacobian, identity z = 0
static_assert(sizeof(G1Affine) == 64 && sizeof(G1) == 96, "layout must match the C ABI");

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error("h2b200 error " + std::to_string(c) + ": " + m), code(c) {}
};

class Context {
public:
    explicit Context(int device = 0) {
        int rc = h2b_ctx_create(device, &ctx_);
        if (rc != H2B_OK) throw Error(rc, h2b_last_error(nullptr));
    }
    // one process, several GPUs (h2b_ctx_create_multi): commitments and batched transforms use all of them
    explicit Context(const std::vector<int>& devices) {
        int rc = h2b_ctx_create_multi(devices.data(), (int)devices.size(), &ctx_);
        if (rc != H2B_OK) throw Error(rc, h2b_last_error(nullptr));
    }
    // a view of a context the caller owns and destroys (a binding that already holds the handle)
    explicit Context(h2b_ctx* borrowed) : ctx_(borrowed), owned_(false) {}
    int device_count() const { return h2b_ctx_device_count(ctx_); }
    ~Context() {
        if (owned_) h2b_ctx_destroy(ctx_);
    }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    h2b_ctx* raw() const { return ctx_; }
    void check(int rc) const {
        if (rc != H2B_OK) throw Error(rc, h2b_last_error(ctx_));
    }
    void set_stream(void* cuda_stream) { check(h2b_ctx_set_stream(ctx_, cuda_stream)); }
    // tuning switches ("msm.batch_group", "ntt.max_ctas_per_sm"; include/h2b200.h): never change a result
    void set_option(const char* key, int64_t value) { check(h2b_ctx_set_option(ctx_, key, value)); }
    void synchronize() { check(h2b_ctx_synchronize(ctx_)); }
    G1 sum(const std::vector<G1>& pts) const {  // combine per-GPU partial commitments
        G1 out;
        check(h2b_g1_sum(ctx_, reinterpret_cast<const uint64_t*>(pts.data()), pts.size(), out.x.data()));
        return out;
    }
    void batch_normalize(std::vector<G1>& pts) const {
        check(h2b_g1_normalize(ctx_, reinterpret_cast<uint64_t*>(pts.data()), pts.size()));
    }

private:
    h2b_ctx* ctx_ = nullptr;
    bool owned_ = true;
};

// best_multiexp(coeffs, bases): ad-hoc bases.  Rust asserts coeffs.len() == bases.len().
inline G1 best_multiexp(const Context& ctx, const std::vector<Fr>& coeffs, const std::vector<G1Affine>& bases) {
    if (coeffs.size() != bases.size()) throw Error(H2B_ERR_ARG, "best_multiexp: coeffs.len() != bases.len()");
    G1 out;
    ctx.check(h2b_msm_g1_bases(ctx.raw(), reinterpret_cast<const uint64_t*>(bases.data()),
                               reinterpret_cast<const uint64_t*>(coeffs.data()), coeffs.size(), out.x.data()));
    return out;
}

// best_fft(a, omega, log_n): in place.
inline void best_fft(const Context& ctx, std::vector<Fr>& a, const Fr& omega, uint32_t log_n) {
    if (a.size() != (size_t(1) << log_n)) throw Error(H2B_ERR_ARG, "best_fft: a.len() != 1 << log_n");
    ctx.check(h2b_ntt_fr(ctx.raw(), reinterpret_cast<uint64_t*>(a.data()), log_n, omega.data(), 0));
}

enum class SerdeFormat { Processed, RawBytes };

namespace detail {
// elems x 32 bytes of device memory (one h2b_poly); an affine G1 point takes two elements
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(const Context& ctx, size_t elems) : ctx_(&ctx) { ctx.check(h2b_poly_alloc(ctx.raw(), elems, &h_)); }
    DeviceBuffer(DeviceBuffer&& o) noexcept : ctx_(o.ctx_), h_(o.h_) { o.h_ = nullptr; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        std::swap(ctx_, o.ctx_);
        std::swap(h_, o.h_);
        return *this;
    }
    ~DeviceBuffer() {
        if (h_) h2b_poly_free(ctx_->raw(), h_);
    }
    void* ptr() const { return h_ ? h2b_poly_device_ptr(h_) : nullptr; }
    h2b_poly* raw() const { return h_; }

private:
    const Context* ctx_ = nullptr;
    h2b_poly* h_ = nullptr;
};
// the G1 generator (1, 2), Montgomery limbs: the base of ParamsKZG::setup
inline const uint64_t* g1_generator() {
    static const uint64_t g[8] = {0xd35d438dc58f0d9dULL, 0x0a78eb28f5c70b3dULL, 0x666ea36f7879462cULL, 0x0e0a77c19a07df2fULL,
                                  0xa6ba871b8b1e1b3aULL, 0x14f1d651eb8e167bULL, 0xccdd46def0f28c58ULL, 0x1c14ef83340fbe5eULL};
    return g;
}
struct ImageView {
    uint32_t k;
    size_t off[4];  // g, g_lagrange, g2, s_g2
};
inline ImageView processed_view(const std::vector<uint8_t>& image) {
    ImageView v{};
    const int rc = h2b_params_processed_view(image.data(), image.size(), &v.k, &v.off[0], &v.off[1], &v.off[2], &v.off[3]);
    if (rc != H2B_OK) throw Error(H2B_ERR_ARG, "read_params: not a SerdeFormat::Processed params image");
    return v;
}
}  // namespace detail

// The base arrays of ParamsKZG<Bn256> resident on one GPU (this rank's shard [begin, begin + count)).
// Params made by setup_seeded / read_downsized (and gen_srs when it creates the file) also keep g and g_lagrange themselves on
// the device, whole, and the G2 pair (g2, s_g2): they can be written (ParamsKZG::write) and downsized (Params::downsize).
class ParamsKZG {
public:
    ParamsKZG(const Context& ctx, uint32_t k, const std::vector<G1Affine>& g, const std::vector<G1Affine>& g_lagrange,
              size_t begin = 0, size_t count = 0)
        : ctx_(ctx), k_(k), count_(count ? count : (size_t(1) << k) - begin) {
        const size_t n = size_t(1) << k;
        if ((!g.empty() && g.size() != n) || (!g_lagrange.empty() && g_lagrange.size() != n))
            throw Error(H2B_ERR_ARG, "ParamsKZG: base arrays must hold 2^k points");
        ctx.check(h2b_srs_upload(ctx.raw(), g.empty() ? nullptr : reinterpret_cast<const uint64_t*>(g.data()),
                                 g_lagrange.empty() ? nullptr : reinterpret_cast<const uint64_t*>(g_lagrange.data()), k,
                                 begin, count_, &srs_));
    }
    // a view of an SRS handle the caller owns and destroys (its shard holds `count` points)
    ParamsKZG(const Context& ctx, uint32_t k, h2b_srs* borrowed, size_t count)
        : ctx_(ctx), k_(k), count_(count), srs_(borrowed), owned_(false) {}
    ~ParamsKZG() {
        if (owned_) h2b_srs_destroy(ctx_.raw(), srs_);
    }
    ParamsKZG(const ParamsKZG&) = delete;
    ParamsKZG& operator=(const ParamsKZG&) = delete;
    ParamsKZG(ParamsKZG&& o) noexcept
        : ctx_(o.ctx_), k_(o.k_), count_(o.count_), srs_(o.srs_), owned_(o.owned_), g_(std::move(o.g_)), gl_(std::move(o.gl_)),
          g2_processed_(std::move(o.g2_processed_)), g2_raw_(std::move(o.g2_raw_)) {
        o.srs_ = nullptr;
    }

    // `ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed))`, what gen_srs creates (seed = 32 zero bytes): g and g_lagrange at
    // halo2-lib's tau on the device, the G2 pair on the host
    static ParamsKZG setup_seeded(const Context& ctx, uint32_t k, const std::array<uint8_t, 32>& seed = {}) {
        Fr tau{};
        if (h2b_srs_seeded_tau(seed.data(), tau.data()) != H2B_OK) throw Error(H2B_ERR_ARG, "setup_seeded: null seed");
        detail::DeviceBuffer g(ctx, size_t(2) << k), gl(ctx, size_t(2) << k);
        ctx.check(h2b_srs_setup_dev(ctx.raw(), tau.data(), detail::g1_generator(), k, g.ptr(), gl.ptr()));
        std::vector<uint8_t> proc(128), raw(256);
        if (h2b_g2_generator_mul(tau.data(), proc.data(), raw.data()) != H2B_OK) throw Error(H2B_ERR_ARG, "setup_seeded: tau");
        return ParamsKZG(ctx, k, std::move(g), std::move(gl), std::move(proc), std::move(raw));
    }
    // `ParamsKZG::read` of a SerdeFormat::Processed image (h2b_srs_read_processed): the SRS handle only, so these params cannot
    // be written or downsized.  Error(H2B_ERR_ARG) for a malformed image or an invalid point encoding.
    static ParamsKZG read(const Context& ctx, const std::vector<uint8_t>& image) {
        const detail::ImageView v = detail::processed_view(image);
        ParamsKZG p(ctx, v.k, nullptr, size_t(1) << v.k);
        p.owned_ = true;
        ctx.check(h2b_srs_read_processed(ctx.raw(), image.data(), image.size(), 0, 0, &p.srs_));
        p.g2_processed_.assign(image.begin() + v.off[2], image.begin() + v.off[2] + 128);
        return p;
    }
    // `read_params(K).downsize(k)` from a SerdeFormat::Processed image: only the first 2^k encodings of g are decompressed on the
    // device, g_lagrange is rebuilt from them and G2 is kept; the 2^K bases never reach the device
    static ParamsKZG read_downsized(const Context& ctx, const std::vector<uint8_t>& image, uint32_t k) {
        const detail::ImageView v = detail::processed_view(image);
        if (k > v.k) throw Error(H2B_ERR_ARG, "downsize: k above the image's k");
        const size_t n = size_t(1) << k;
        detail::DeviceBuffer enc(ctx, n), g(ctx, 2 * n), gl(ctx, 2 * n);
        ctx.check(h2b_poly_upload(ctx.raw(), enc.raw(), 0, reinterpret_cast<const uint64_t*>(image.data() + v.off[0]), n));
        size_t bad = 0;
        ctx.check(h2b_g1_decompress_dev(ctx.raw(), enc.ptr(), n, g.ptr(), &bad));
        if (bad) throw Error(H2B_ERR_ARG, "read_params: the params image holds an invalid G1 encoding");
        ctx.check(h2b_g_to_lagrange_dev(ctx.raw(), g.ptr(), k, gl.ptr()));
        return ParamsKZG(ctx, k, std::move(g), std::move(gl), std::vector<uint8_t>(image.begin() + v.off[2], image.begin() + v.off[2] + 128), {});
    }
    // `ParamsKZG::write`: u32 LE k | g | g_lagrange | g2 | s_g2
    std::vector<uint8_t> write(SerdeFormat format = SerdeFormat::Processed) const {
        need_bases("write");
        const bool proc = format == SerdeFormat::Processed;
        const std::vector<uint8_t>& g2 = proc ? g2_processed_ : g2_raw_;
        if (g2.empty()) throw Error(H2B_ERR_ARG, "write: the G2 encoding of this format is not known for params read from an image");
        auto fn = proc ? h2b_params_write_processed : h2b_params_write_raw;
        size_t len = 0;
        ctx_.check(fn(ctx_.raw(), nullptr, nullptr, k_, nullptr, nullptr, &len));
        std::vector<uint8_t> out(len);
        ctx_.check(fn(ctx_.raw(), g_.ptr(), gl_.ptr(), k_, g2.data(), out.data(), &len));
        return out;
    }
    // `Params::downsize(k)` in place: g keeps its first 2^k points, g_lagrange is rebuilt from them (g_to_lagrange), G2 stays
    void downsize(uint32_t k) {
        need_bases("downsize");
        if (k > k_) throw Error(H2B_ERR_ARG, "downsize: k above the params' k");
        const size_t n = size_t(1) << k;
        detail::DeviceBuffer g(ctx_, 2 * n), gl(ctx_, 2 * n);
        ctx_.check(h2b_poly_copy_dev(ctx_.raw(), g.ptr(), g_.ptr(), 2 * n));
        ctx_.check(h2b_g_to_lagrange_dev(ctx_.raw(), g.ptr(), k, gl.ptr()));
        h2b_srs* srs = nullptr;
        ctx_.check(h2b_srs_upload_dev(ctx_.raw(), g.ptr(), gl.ptr(), k, 0, n, &srs));
        if (owned_) h2b_srs_destroy(ctx_.raw(), srs_);
        srs_ = srs;
        owned_ = true;
        g_ = std::move(g);
        gl_ = std::move(gl);
        k_ = k;
        count_ = n;
    }
    // the whole bases on the device (2^k x 8 limbs each), null for params that do not keep them
    const void* g_dev() const { return g_.ptr(); }
    const void* g_lagrange_dev() const { return gl_.ptr(); }
    const std::vector<uint8_t>& g2_processed() const { return g2_processed_; }  // g2 | s_g2, 64 bytes each
    uint32_t k() const { return k_; }
    const h2b_srs* raw() const { return srs_; }  // for the `_dev` entry points (the resident prover, h2b200_prover.hpp)
    // ParamsKZG::commit(poly in coefficient form) / commit_lagrange(poly in Lagrange form)
    G1 commit(const std::vector<Fr>& poly) const { return commit_(H2B_BASIS_MONOMIAL, poly); }
    G1 commit_lagrange(const std::vector<Fr>& poly) const { return commit_(H2B_BASIS_LAGRANGE, poly); }
    // all independent commitments of one prover phase at once (basis per column: 0 monomial, 1 lagrange)
    std::vector<G1> commit_many(const std::vector<int>& basis, const std::vector<const std::vector<Fr>*>& polys) const {
        if (basis.size() != polys.size()) throw Error(H2B_ERR_ARG, "commit_many: basis.len() != polys.len()");
        std::vector<const uint64_t*> ptrs;
        for (auto* p : polys) {
            if (!p || p->size() != count_) throw Error(H2B_ERR_ARG, "commit_many: polynomial length != shard size");
            ptrs.push_back(reinterpret_cast<const uint64_t*>(p->data()));
        }
        std::vector<G1> out(polys.size());
        ctx_.check(h2b_msm_g1_batch(ctx_.raw(), srs_, basis.data(), ptrs.data(), polys.size(), count_,
                                    reinterpret_cast<uint64_t*>(out.data())));
        return out;
    }

private:
    ParamsKZG(const Context& ctx, uint32_t k, detail::DeviceBuffer g, detail::DeviceBuffer gl, std::vector<uint8_t> g2_processed,
              std::vector<uint8_t> g2_raw)
        : ctx_(ctx), k_(k), count_(size_t(1) << k), g_(std::move(g)), gl_(std::move(gl)), g2_processed_(std::move(g2_processed)),
          g2_raw_(std::move(g2_raw)) {
        ctx.check(h2b_srs_upload_dev(ctx.raw(), g_.ptr(), gl_.ptr(), k, 0, count_, &srs_));
    }
    void need_bases(const char* what) const {
        if (!g_.ptr()) throw Error(H2B_ERR_ARG, std::string(what) + ": these params do not keep their bases on the device");
    }
    G1 commit_(int basis, const std::vector<Fr>& poly) const {
        G1 out;
        ctx_.check(h2b_msm_g1(ctx_.raw(), srs_, basis, reinterpret_cast<const uint64_t*>(poly.data()), poly.size(), out.x.data()));
        return out;
    }
    const Context& ctx_;
    uint32_t k_;
    size_t count_;
    h2b_srs* srs_ = nullptr;
    bool owned_ = true;
    detail::DeviceBuffer g_, gl_;
    std::vector<uint8_t> g2_processed_, g2_raw_;
};

// where gen_srs caches the params of 2^k rows: dir (default $PARAMS_DIR, else ./params) / kzg_bn254_{k}.srs
inline std::string srs_path(uint32_t k, std::string dir = "") {
    if (dir.empty()) {
        const char* env = std::getenv("PARAMS_DIR");
        dir = env ? env : "./params";
    }
    return dir + "/kzg_bn254_" + std::to_string(k) + ".srs";
}
// halo2-base `gen_srs(k)` = read_or_create_srs: read the cached SerdeFormat::Processed params when the file exists
// (ParamsKZG::read), else create them (setup_seeded, zero seed), create the directory and write the file
inline ParamsKZG gen_srs(const Context& ctx, uint32_t k, const std::string& dir = "") {
    const std::string path = srs_path(k, dir);
    std::ifstream in(path, std::ios::binary);
    if (in) {
        std::vector<uint8_t> image((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
        return ParamsKZG::read(ctx, image);
    }
    ParamsKZG params = ParamsKZG::setup_seeded(ctx, k);
    const std::vector<uint8_t> image = params.write(SerdeFormat::Processed);
    std::filesystem::create_directories(std::filesystem::path(path).parent_path());
    std::ofstream out(path, std::ios::binary);
    out.write(reinterpret_cast<const char*>(image.data()), std::streamsize(image.size()));
    if (!out) throw Error(H2B_ERR_ARG, "gen_srs: cannot write " + path);
    return params;
}

// EvaluationDomain::new(j, k): j = cs.degree(); quotient_poly_degree = j - 1; extended_k = least e >= k with
// 2^e >= n * (j - 1) (SURVEY.md Appendix B).
class EvaluationDomain {
public:
    EvaluationDomain(const Context& ctx, uint32_t j, uint32_t k) : ctx_(ctx), k_(k), quotient_poly_degree_(j - 1) {
        extended_k_ = k;
        while ((uint64_t(1) << extended_k_) < (uint64_t(1) << k) * quotient_poly_degree_) extended_k_++;
        ctx.check(h2b_domain_omega(k, omega_.data()));
    }
    uint32_t k() const { return k_; }
    uint32_t extended_k() const { return extended_k_; }
    const Fr& get_omega() const { return omega_; }
    void lagrange_to_coeff(std::vector<Fr>& a) const {
        expect(a.size() == n(), "lagrange_to_coeff: a.len() != n");
        ctx_.check(h2b_lagrange_to_coeff(ctx_.raw(), reinterpret_cast<uint64_t*>(a.data()), k_));
    }
    void coeff_to_lagrange(std::vector<Fr>& a) const {
        expect(a.size() == n(), "coeff_to_lagrange: a.len() != n");
        ctx_.check(h2b_coeff_to_lagrange(ctx_.raw(), reinterpret_cast<uint64_t*>(a.data()), k_));
    }
    std::vector<Fr> coeff_to_extended(const std::vector<Fr>& a) const {
        expect(a.size() == n(), "coeff_to_extended: a.len() != n");
        std::vector<Fr> out(size_t(1) << extended_k_);
        ctx_.check(h2b_coeff_to_extended(ctx_.raw(), reinterpret_cast<const uint64_t*>(a.data()), a.size(), extended_k_,
                                         reinterpret_cast<uint64_t*>(out.data())));
        return out;
    }
    std::vector<Fr> extended_to_coeff(std::vector<Fr> a) const {
        expect(a.size() == (size_t(1) << extended_k_), "extended_to_coeff: a.len() != extended_len");
        ctx_.check(h2b_extended_to_coeff(ctx_.raw(), reinterpret_cast<uint64_t*>(a.data()), extended_k_));
        a.resize(n() * quotient_poly_degree_);  // `a.values.truncate(n * quotient_poly_degree)`
        return a;
    }

private:
    size_t n() const { return size_t(1) << k_; }
    static void expect(bool ok, const char* msg) {
        if (!ok) throw Error(H2B_ERR_ARG, msg);
    }
    const Context& ctx_;
    uint32_t k_, extended_k_ = 0;
    uint64_t quotient_poly_degree_;
    Fr omega_{};
};

// assign_witnesses(threads, basic_gates, region, break_points): `threads[i]` = ctx.advice of the i-th Context
// (Trivial payloads); returns basic_gates.len() columns of 2^k rows.  Throws h2b::Error(H2B_ERR_LAYOUT) where Rust panics.
inline std::vector<std::vector<Fr>> assign_witnesses(const Context& ctx, const std::vector<std::vector<Fr>>& threads,
                                                     const std::vector<uint64_t>& break_points, uint32_t k, size_t num_columns) {
    std::vector<Fr> vcol;
    for (auto& t : threads) vcol.insert(vcol.end(), t.begin(), t.end());
    std::vector<Fr> flat(num_columns << k);
    ctx.check(h2b_assign_columns(ctx.raw(), reinterpret_cast<const uint64_t*>(vcol.data()), vcol.size(), break_points.data(),
                                 break_points.size(), k, num_columns, reinterpret_cast<uint64_t*>(flat.data())));
    std::vector<std::vector<Fr>> cols(num_columns);
    for (size_t c = 0; c < num_columns; c++) cols[c].assign(flat.begin() + (c << k), flat.begin() + ((c + 1) << k));
    return cols;
}

// LookupAnyManager::assign_raw: value j -> lookup column j % L, row j / L
inline std::vector<std::vector<Fr>> assign_lookups(const Context& ctx, const std::vector<Fr>& values, uint32_t k, size_t L) {
    std::vector<Fr> flat(L << k);
    ctx.check(h2b_assign_lookups(ctx.raw(), reinterpret_cast<const uint64_t*>(values.data()), values.size(), k, L,
                                 reinterpret_cast<uint64_t*>(flat.data())));
    std::vector<std::vector<Fr>> cols(L);
    for (size_t c = 0; c < L; c++) cols[c].assign(flat.begin() + (c << k), flat.begin() + ((c + 1) << k));
    return cols;
}

// halo2-base's own witness form on the device (asynchronous, device pointers; see h2b200.h): batch_invert_assigned of the
// Rational cells in place, and assign_raw from virtual-column indices.  Violations land in the device word *d_status.
inline void apply_rational_dev(const Context& ctx, void* d_values, size_t N, const void* d_index, void* d_den, size_t R, uint32_t* d_status) {
    ctx.check(h2b_apply_rational_dev(ctx.raw(), d_values, N, d_index, d_den, R, d_status));
}
inline void assign_lookups_indexed_dev(const Context& ctx, const void* d_values, size_t N, const void* d_index, size_t n_lookup, uint32_t k,
                                       size_t L, void* d_cols, uint32_t* d_status) {
    ctx.check(h2b_assign_lookups_indexed_dev(ctx.raw(), d_values, N, d_index, n_lookup, k, L, d_cols, d_status));
}

// the constraint check (asynchronous, device pointers; see h2b200.h): reports of max_report + 1 u64 words per checked item
inline void check_graph_dev(const Context& ctx, const h2b_graph& g, uint32_t k, size_t rows, size_t max_report, void* d_report) {
    ctx.check(h2b_check_graph_dev(ctx.raw(), &g, k, rows, max_report, d_report));
}
inline void check_lookup_dev(const Context& ctx, const void* d_input, const void* d_table, uint32_t k, size_t rows, size_t max_report,
                             void* d_report) {
    ctx.check(h2b_check_lookup_dev(ctx.raw(), d_input, d_table, k, rows, max_report, d_report));
}
inline void permutation_decode_dev(const Context& ctx, const std::vector<const void*>& d_sigma, uint32_t k, void* d_map, size_t max_report,
                                   void* d_reports) {
    ctx.check(h2b_permutation_decode_dev(ctx.raw(), d_sigma.data(), d_sigma.size(), k, d_map, max_report, d_reports));
}
inline void check_copies_dev(const Context& ctx, const std::vector<const void*>& d_columns, const void* d_map, uint32_t k, size_t max_report,
                             void* d_reports) {
    ctx.check(h2b_check_copies_dev(ctx.raw(), d_columns.data(), d_map, d_columns.size(), k, max_report, d_reports));
}

// arithmetic::eval_polynomial(poly, point)
inline Fr eval_polynomial(const Context& ctx, const std::vector<Fr>& poly, const Fr& point) {
    Fr out{};
    ctx.check(h2b_eval_polynomial(ctx.raw(), reinterpret_cast<const uint64_t*>(poly.data()), poly.size(),
                                  reinterpret_cast<const uint64_t*>(&point), reinterpret_cast<uint64_t*>(&out)));
    return out;
}

// arithmetic::kate_division(a, b): quotient of a(X) by (X - b), remainder dropped
inline std::vector<Fr> kate_division(const Context& ctx, const std::vector<Fr>& a, const Fr& b) {
    std::vector<Fr> q(a.empty() ? 0 : a.size() - 1);
    ctx.check(h2b_kate_division(ctx.raw(), reinterpret_cast<const uint64_t*>(a.data()), a.size(), reinterpret_cast<const uint64_t*>(&b),
                                reinterpret_cast<uint64_t*>(q.data())));
    return q;
}

// ff::BatchInvert::batch_invert on a slice (zeros stay zero)
inline void batch_invert(const Context& ctx, std::vector<Fr>& a) {
    ctx.check(h2b_batch_invert_fr(ctx.raw(), reinterpret_cast<uint64_t*>(a.data()), a.size()));
}
// z[0] = start, z[i] = z[i-1] * f[i-1]
inline std::vector<Fr> grand_product(const Context& ctx, const std::vector<Fr>& f, const Fr& start) {
    std::vector<Fr> z(f.size());
    ctx.check(h2b_grand_product_fr(ctx.raw(), reinterpret_cast<const uint64_t*>(f.data()), start.data(), f.size(),
                                   reinterpret_cast<uint64_t*>(z.data())));
    return z;
}
// permute_expression_pair: (A', S') over the usable rows, the last blinding_factors + 1 rows left zero for the caller's
// blinding scalars.  Throws Error(H2B_ERR_UNSATISFIED) for `Error::ConstraintSystemFailure`.
inline std::pair<std::vector<Fr>, std::vector<Fr>> permute_expression_pair(const Context& ctx, const std::vector<Fr>& input,
                                                                           const std::vector<Fr>& table, uint32_t k,
                                                                           uint32_t blinding_factors) {
    if (input.size() != (size_t(1) << k) || table.size() != input.size()) throw Error(H2B_ERR_ARG, "permute_expression_pair: need 2^k rows");
    std::vector<Fr> a(input.size(), Fr{0, 0, 0, 0}), s(input.size(), Fr{0, 0, 0, 0});
    ctx.check(h2b_permute_expression_pair(ctx.raw(), reinterpret_cast<const uint64_t*>(input.data()),
                                          reinterpret_cast<const uint64_t*>(table.data()), k, blinding_factors,
                                          reinterpret_cast<uint64_t*>(a.data()), reinterpret_cast<uint64_t*>(s.data())));
    return {a, s};
}

// ---- plonk::evaluation::GraphEvaluator: value sources, calculations, and the program h2b_graph carries
struct ValueSource {
    uint32_t kind, index, rotation_slot;
    static ValueSource Constant(uint32_t i) { return {H2B_SRC_CONSTANT, i, 0}; }
    static ValueSource Intermediate(uint32_t i) { return {H2B_SRC_INTERMEDIATE, i, 0}; }
    static ValueSource Fixed(uint32_t col, uint32_t rot) { return {H2B_SRC_FIXED, col, rot}; }
    static ValueSource Advice(uint32_t col, uint32_t rot) { return {H2B_SRC_ADVICE, col, rot}; }
    static ValueSource Instance(uint32_t col, uint32_t rot) { return {H2B_SRC_INSTANCE, col, rot}; }
    static ValueSource Challenge(uint32_t i) { return {H2B_SRC_CHALLENGE, i, 0}; }
    static ValueSource Beta() { return {H2B_SRC_BETA, 0, 0}; }
    static ValueSource Gamma() { return {H2B_SRC_GAMMA, 0, 0}; }
    static ValueSource Theta() { return {H2B_SRC_THETA, 0, 0}; }
    static ValueSource Y() { return {H2B_SRC_Y, 0, 0}; }
    static ValueSource PreviousValue() { return {H2B_SRC_PREVIOUS, 0, 0}; }
    uint32_t word() const { return H2B_SRC(kind, index, rotation_slot); }
    bool operator==(const ValueSource& o) const { return kind == o.kind && index == o.index && rotation_slot == o.rotation_slot; }
};
struct Calculation {
    uint32_t op;                     // H2B_CALC_*
    std::vector<ValueSource> args;   // Horner: start, factor, parts...
    static Calculation Add(ValueSource a, ValueSource b) { return {H2B_CALC_ADD, {a, b}}; }
    static Calculation Sub(ValueSource a, ValueSource b) { return {H2B_CALC_SUB, {a, b}}; }
    static Calculation Mul(ValueSource a, ValueSource b) { return {H2B_CALC_MUL, {a, b}}; }
    static Calculation Square(ValueSource a) { return {H2B_CALC_SQUARE, {a}}; }
    static Calculation Double(ValueSource a) { return {H2B_CALC_DOUBLE, {a}}; }
    static Calculation Negate(ValueSource a) { return {H2B_CALC_NEGATE, {a}}; }
    static Calculation Store(ValueSource a) { return {H2B_CALC_STORE, {a}}; }
    static Calculation Horner(ValueSource start, std::vector<ValueSource> parts, ValueSource factor) {
        std::vector<ValueSource> v{start, factor};
        v.insert(v.end(), parts.begin(), parts.end());
        return {H2B_CALC_HORNER, v};
    }
    bool operator==(const Calculation& o) const { return op == o.op && args == o.args; }
};
class GraphEvaluator {
public:
    uint32_t add_rotation(int32_t rotation) {
        auto it = std::find(rotations.begin(), rotations.end(), rotation);
        if (it != rotations.end()) return uint32_t(it - rotations.begin());
        rotations.push_back(rotation);
        return uint32_t(rotations.size() - 1);
    }
    ValueSource add_constant(const Fr& c) {
        auto it = std::find(constants.begin(), constants.end(), c);
        if (it != constants.end()) return ValueSource::Constant(uint32_t(it - constants.begin()));
        constants.push_back(c);
        return ValueSource::Constant(uint32_t(constants.size() - 1));
    }
    ValueSource add_calculation(const Calculation& c) {  // identical calculations are shared, as upstream does
        auto it = std::find(calculations.begin(), calculations.end(), c);
        if (it != calculations.end()) return ValueSource::Intermediate(uint32_t(it - calculations.begin()));
        calculations.push_back(c);
        return ValueSource::Intermediate(uint32_t(calculations.size() - 1));
    }
    std::vector<uint32_t> program() const {
        std::vector<uint32_t> w;
        for (auto& c : calculations) {
            w.push_back(c.op);
            if (c.op == H2B_CALC_HORNER) {
                w.push_back(c.args[0].word());
                w.push_back(c.args[1].word());
                w.push_back(uint32_t(c.args.size() - 2));
                for (size_t j = 2; j < c.args.size(); j++) w.push_back(c.args[j].word());
            } else {
                for (auto& a : c.args) w.push_back(a.word());
            }
        }
        return w;
    }
    std::vector<Fr> constants;
    std::vector<int32_t> rotations;
    std::vector<Calculation> calculations;
};
struct Challenges {
    Fr beta{}, gamma{}, theta{}, y{};
    std::vector<Fr> user;  // ValueSource::Challenge(i)
};
// an h2b_graph together with the arrays it points to (the program words, the column tables, the user challenges): valid while
// the value lives.  The column tables hold host or device pointers, as the entry point the graph goes to takes them.
class BoundGraph {
public:
    BoundGraph(const GraphEvaluator& ev, ValueSource result, std::vector<const void*> fixed, std::vector<const void*> advice,
               const Challenges& ch = {}, std::vector<const void*> instance = {})
        : prog_(ev.program()), fixed_(std::move(fixed)), advice_(std::move(advice)), instance_(std::move(instance)), user_(ch.user) {
        g_.program = prog_.data();
        g_.program_words = prog_.size();
        g_.n_calculations = uint32_t(ev.calculations.size());
        g_.result = result.word();
        g_.constants = reinterpret_cast<const uint64_t*>(ev.constants.data());
        g_.n_constants = ev.constants.size();
        g_.rotations = ev.rotations.data();
        g_.n_rotations = ev.rotations.size();
        g_.fixed = fixed_.data();
        g_.n_fixed = fixed_.size();
        g_.advice = advice_.data();
        g_.n_advice = advice_.size();
        g_.instance = instance_.data();
        g_.n_instance = instance_.size();
        g_.challenges = reinterpret_cast<const uint64_t*>(user_.data());
        g_.n_challenges = user_.size();
        std::copy(ch.beta.begin(), ch.beta.end(), g_.beta);
        std::copy(ch.gamma.begin(), ch.gamma.end(), g_.gamma);
        std::copy(ch.theta.begin(), ch.theta.end(), g_.theta);
        std::copy(ch.y.begin(), ch.y.end(), g_.y);
    }
    BoundGraph(const BoundGraph&) = delete;
    BoundGraph& operator=(const BoundGraph&) = delete;
    const h2b_graph* get() const { return &g_; }

private:
    std::vector<uint32_t> prog_;
    std::vector<const void*> fixed_, advice_, instance_;
    std::vector<Fr> user_;
    h2b_graph g_{};
};

using Columns = std::vector<const std::vector<Fr>*>;  // extended-domain columns (2^ext_k values each)
namespace detail {
inline std::vector<const void*> tables(const Columns& cols) {
    std::vector<const void*> p;
    for (auto c : cols) p.push_back(c->data());
    return p;
}
inline std::vector<const uint64_t*> ptrs(const Columns& cols) {
    std::vector<const uint64_t*> p;
    for (auto c : cols) p.push_back(reinterpret_cast<const uint64_t*>(c->data()));
    return p;
}
}  // namespace detail

// custom gates of evaluate_h: values[i] = graph(previous = values[i]) on every extended-domain row
inline void quotient_graph(const Context& ctx, const GraphEvaluator& ev, ValueSource result, const Columns& fixed, const Columns& advice,
                           const Columns& instance, const Challenges& ch, uint32_t k, uint32_t ext_k, std::vector<Fr>& values) {
    const BoundGraph g(ev, result, detail::tables(fixed), detail::tables(advice), ch, detail::tables(instance));
    ctx.check(h2b_quotient_graph(ctx.raw(), g.get(), k, ext_k, reinterpret_cast<uint64_t*>(values.data())));
}
inline void permutation_fold(const Context& ctx, const Columns& z_sets, const Columns& columns, const Columns& sigma, size_t chunk_len,
                             const std::vector<Fr>& l0, const std::vector<Fr>& l_last, const std::vector<Fr>& l_active,
                             const Challenges& ch, uint32_t blinding_factors, uint32_t k, uint32_t ext_k, std::vector<Fr>& values) {
    auto z = detail::ptrs(z_sets), c = detail::ptrs(columns), s = detail::ptrs(sigma);
    ctx.check(h2b_permutation_fold(ctx.raw(), z.data(), z.size(), c.data(), s.data(), c.size(), chunk_len,
                                   reinterpret_cast<const uint64_t*>(l0.data()), reinterpret_cast<const uint64_t*>(l_last.data()),
                                   reinterpret_cast<const uint64_t*>(l_active.data()), ch.beta.data(), ch.gamma.data(), ch.y.data(),
                                   blinding_factors, k, ext_k, reinterpret_cast<uint64_t*>(values.data())));
}
inline void lookup_fold(const Context& ctx, const GraphEvaluator& ev, ValueSource result, const Columns& fixed, const Columns& advice,
                        const Columns& instance, const Challenges& ch, const std::vector<Fr>& z, const std::vector<Fr>& permuted_input,
                        const std::vector<Fr>& permuted_table, const std::vector<Fr>& l0, const std::vector<Fr>& l_last,
                        const std::vector<Fr>& l_active, uint32_t k, uint32_t ext_k, std::vector<Fr>& values) {
    const BoundGraph g(ev, result, detail::tables(fixed), detail::tables(advice), ch, detail::tables(instance));
    auto p = [](const std::vector<Fr>& v) { return reinterpret_cast<const uint64_t*>(v.data()); };
    ctx.check(h2b_lookup_fold(ctx.raw(), g.get(), p(z), p(permuted_input), p(permuted_table), p(l0), p(l_last), p(l_active), k, ext_k,
                              reinterpret_cast<uint64_t*>(values.data())));
}
inline void divide_by_vanishing_poly(const Context& ctx, std::vector<Fr>& values, uint32_t k, uint32_t ext_k) {
    ctx.check(h2b_divide_by_vanishing_poly(ctx.raw(), reinterpret_cast<uint64_t*>(values.data()), k, ext_k));
}
// poly::kzg::commitment::g_to_lagrange
inline std::vector<G1Affine> g_to_lagrange(const Context& ctx, const std::vector<G1Affine>& g, uint32_t k) {
    if (g.size() != (size_t(1) << k)) throw Error(H2B_ERR_ARG, "g_to_lagrange: need 2^k points");
    std::vector<G1Affine> out(g.size());
    ctx.check(h2b_g_to_lagrange(ctx.raw(), reinterpret_cast<const uint64_t*>(g.data()), k, reinterpret_cast<uint64_t*>(out.data())));
    return out;
}

}  // namespace h2b
