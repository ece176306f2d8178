// prover.cu — device-resident polynomials and the product columns of create_proof's permutation / lookup arguments.
//
// halo2-axiom 0.5.3 keeps every column of a proof as a `Polynomial<Fr, _>` on the host and walks them with rayon
// (plonk/prover.rs, plonk/permutation/prover.rs `commit`, plonk/lookup/prover.rs `commit_product`; not vendored —
// restated from the protocol, parity unpinned like the rest of L0; reached from the one create_proof call site
// halo2-base/src/utils/testing.rs:40-48).  Here a column lives in HBM behind an opaque `h2b_poly` handle from the
// moment it is assigned or computed until the proof is finished; only commitments, evaluations and blinding scalars
// cross PCIe.  Every `_dev` entry point of the library accepts `h2b_poly_device_ptr()`.
//
//   h2b_permutation_product_dev   z[0] = start, z[i+1] = z[i] * prod_j (v_j + beta delta^j omega^i + gamma)
//                                                             / prod_j (v_j + beta sigma_j(i) + gamma)      (i < u)
//   h2b_lookup_product_dev        z[0] = 1,     z[i+1] = z[i] * (a_i + beta)(s_i + gamma) / ((a'_i + beta)(s'_i + gamma))
//   h2b_fr_mul_elementwise_dev    compressed lookup input q * a (halo2-base/src/gates/range/mod.rs:131-140)
//   h2b_eval_polynomial_batch_dev the evaluations create_proof writes to the transcript after the challenge x
// u = 2^k - (blinding_factors + 1) usable rows; rows above u are left to the caller's blinding scalars.
#include <cstring>

#include "h2b_internal.cuh"
#include "field.cuh"
#include "fr_domain_consts.inc"

struct h2b_poly {
    void* p = nullptr;
    size_t n = 0;
    int device = 0;
};

namespace h2b {

static Fr fr_of_limbs(const uint64_t x[4]) {
    Fr r;
    memcpy(&r, x, sizeof(Fr));
    return r;
}

static constexpr int PP_MAX_COLS = 8;
struct PermProdArgs {
    const uint64_t* cols[PP_MAX_COLS];
    const uint64_t* sigma[PP_MAX_COLS];
    const uint64_t* pow_lo;  // [i] = omega^i, i < 2^lo_bits
    const uint64_t* pow_hi;  // [j] = beta * delta^first_col * omega^(j << lo_bits)
    u32 n_cols, lo_bits;
    Fr beta, gamma, delta;
};
struct OmegaPow2 {
    Fr w[28];  // omega^(2^j) of the 2^k domain
};

__global__ void __launch_bounds__(256) k_pp_tables(OmegaPow2 ow, u32 k, u32 lo_bits, Fr hi_scale, uint64_t* __restrict__ lo,
                                                   uint64_t* __restrict__ hi) {
    const u32 idx = blockIdx.x * blockDim.x + threadIdx.x, n_lo = 1u << lo_bits, hi_bits = k - lo_bits;
    if (idx < n_lo) {
        Fr r = Fr::one();
        for (u32 j = 0; j < lo_bits; j++)
            if ((idx >> j) & 1) r = r * ow.w[j];
        r.store(lo + 4 * (size_t)idx);
    } else if (idx - n_lo < (1u << hi_bits)) {
        const u32 h = idx - n_lo;
        Fr r = hi_scale;
        for (u32 j = 0; j < hi_bits; j++)
            if ((h >> j) & 1) r = r * ow.w[lo_bits + j];
        r.store(hi + 4 * (size_t)h);
    }
}

// hi[i] *= delta^e (every thread recomputes the small power: e is a column index)
__global__ void __launch_bounds__(256) k_pp_scale_hi(uint64_t* __restrict__ hi, size_t n_hi, Fr delta, u32 e) {
    Fr s = Fr::one(), b = delta;
    for (u32 x = e; x; x >>= 1) {
        if (x & 1) s = s * b;
        b = b.sqr();
    }
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_hi) (Fr::load(hi + 4 * i) * s).store(hi + 4 * i);
}

// numerator / denominator of the permutation product's row factor (1 on the rows that are not usable)
__global__ void __launch_bounds__(256) k_perm_terms(PermProdArgs a, size_t u, size_t n, uint64_t* __restrict__ num,
                                                    uint64_t* __restrict__ den) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr nu = Fr::one(), de = Fr::one();
    if (i < u) {
        Fr cur = Fr::load_nc(a.pow_hi + 4 * (i >> a.lo_bits)) * Fr::load_nc(a.pow_lo + 4 * (i & (((size_t)1 << a.lo_bits) - 1)));
#pragma unroll 1
        for (u32 j = 0; j < a.n_cols; j++) {
            const Fr v = Fr::load_nc(a.cols[j] + 4 * i);
            nu = nu * (v + cur + a.gamma);
            de = de * (v + a.beta * Fr::load_nc(a.sigma[j] + 4 * i) + a.gamma);
            cur = cur * a.delta;
        }
    }
    nu.store(num + 4 * i);
    de.store(den + 4 * i);
}

__global__ void __launch_bounds__(256) k_lookup_terms(const uint64_t* __restrict__ in, const uint64_t* __restrict__ tab,
                                                      const uint64_t* __restrict__ pin, const uint64_t* __restrict__ ptab, Fr beta,
                                                      Fr gamma, size_t u, size_t n, uint64_t* __restrict__ num, uint64_t* __restrict__ den) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr nu = Fr::one(), de = Fr::one();
    if (i < u) {
        nu = (Fr::load_nc(in + 4 * i) + beta) * (Fr::load_nc(tab + 4 * i) + gamma);
        de = (Fr::load_nc(pin + 4 * i) + beta) * (Fr::load_nc(ptab + 4 * i) + gamma);
    }
    nu.store(num + 4 * i);
    de.store(den + 4 * i);
}

__global__ void __launch_bounds__(256) k_fr_mul(const uint64_t* x, const uint64_t* y, size_t n, uint64_t* out) {  // out may alias x
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    (Fr::load(x + 4 * i) * Fr::load(y + 4 * i)).store(out + 4 * i);
}

// z from the row factors num / den:  den <- 1/den (batch), f = num * den, z = prefix products seeded with `start`
static void product_column(h2b_ctx* ctx, uint64_t* num, uint64_t* den, size_t n, const void* d_start, void* d_z) {
    batch_invert_run(ctx, den, n);
    H2B_LAUNCH(ctx, k_fr_mul, ceil_div(n, 256), 256, 0, (const uint64_t*)num, (const uint64_t*)den, n, num);
    uint64_t one[4];
    for (int i = 0; i < 4; i++) one[i] = ((uint64_t)FrParams::ONE(2 * i + 1) << 32) | FrParams::ONE(2 * i);
    grand_product_run(ctx, num, one, n, d_z, d_start);
}

void permutation_product_run(h2b_ctx* ctx, const void* const* d_columns, const void* const* d_sigma, size_t n_cols, size_t first_col,
                             const uint64_t beta[4], const uint64_t gamma[4], uint32_t k, uint32_t blinding_factors,
                             const void* d_start, void* d_z) {
    H2B_REQUIRE(k >= 1 && k <= 27, "permutation_product: k out of range");
    H2B_REQUIRE(n_cols >= 1 && n_cols <= (size_t)PP_MAX_COLS, "permutation_product: 1..8 columns per set");
    const size_t n = (size_t)1 << k;
    H2B_REQUIRE((size_t)blinding_factors + 1 < n, "permutation_product: no usable rows");
    const size_t u = n - (blinding_factors + 1);
    PermProdArgs a;
    memset(&a, 0, sizeof(a));
    for (size_t j = 0; j < n_cols; j++) {
        H2B_REQUIRE(d_columns[j] && d_sigma[j], "permutation_product: null column");
        a.cols[j] = (const uint64_t*)d_columns[j];
        a.sigma[j] = (const uint64_t*)d_sigma[j];
    }
    a.n_cols = (u32)n_cols;
    a.beta = fr_of_limbs(beta);
    a.gamma = fr_of_limbs(gamma);
    a.delta = fr_of_limbs(FR_DELTA_U64);
    a.lo_bits = k < 10 ? k : 10;
    const size_t n_lo = (size_t)1 << a.lo_bits, n_hi = (size_t)1 << (k - a.lo_bits);
    // scratch: power tables, numerators, denominators
    uint64_t* ws = (uint64_t*)ctx->get(WS_PROD, 32 * (n_lo + n_hi + 2 * n));
    uint64_t *lo = ws, *hi = ws + 4 * n_lo, *num = hi + 4 * n_hi, *den = num + 4 * n;
    a.pow_lo = lo;
    a.pow_hi = hi;
    OmegaPow2 ow;
    for (uint32_t j = 0; j < k; j++) memcpy(&ow.w[j], FR_OMEGA[k - j], 32);  // omega^(2^j) = omega_{k - j}
    // hi table = beta * omega^(j << lo_bits), then scaled by delta^first_col (the set's first column index)
    H2B_LAUNCH(ctx, k_pp_tables, ceil_div(n_lo + n_hi, 256), 256, 0, ow, k, a.lo_bits, a.beta, lo, hi);
    if (first_col) H2B_LAUNCH(ctx, k_pp_scale_hi, ceil_div(n_hi, 256), 256, 0, hi, n_hi, a.delta, (u32)first_col);
    H2B_LAUNCH(ctx, k_perm_terms, ceil_div(n, 256), 256, 0, a, u, n, num, den);
    product_column(ctx, num, den, n, d_start, d_z);
}

void lookup_product_run(h2b_ctx* ctx, const void* d_in, const void* d_tab, const void* d_pin, const void* d_ptab, const uint64_t beta[4],
                        const uint64_t gamma[4], uint32_t k, uint32_t blinding_factors, void* d_z) {
    H2B_REQUIRE(k >= 1 && k <= 27, "lookup_product: k out of range");
    const size_t n = (size_t)1 << k;
    H2B_REQUIRE((size_t)blinding_factors + 1 < n, "lookup_product: no usable rows");
    const size_t u = n - (blinding_factors + 1);
    uint64_t* ws = (uint64_t*)ctx->get(WS_PROD, 32 * 2 * n);
    uint64_t *num = ws, *den = ws + 4 * n;
    H2B_LAUNCH(ctx, k_lookup_terms, ceil_div(n, 256), 256, 0, (const uint64_t*)d_in, (const uint64_t*)d_tab, (const uint64_t*)d_pin,
               (const uint64_t*)d_ptab, fr_of_limbs(beta), fr_of_limbs(gamma), u, n, num, den);
    product_column(ctx, num, den, n, nullptr, d_z);
}

void fr_mul_elementwise_run(h2b_ctx* ctx, const void* d_a, const void* d_b, size_t n, void* d_out) {
    if (n == 0) return;
    H2B_LAUNCH(ctx, k_fr_mul, ceil_div(n, 256), 256, 0, (const uint64_t*)d_a, (const uint64_t*)d_b, n, (uint64_t*)d_out);
}

}  // namespace h2b

using namespace h2b;

extern "C" {

int h2b_poly_alloc(h2b_ctx* ctx, size_t n_elems, h2b_poly** out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(out, "poly_alloc: null output handle");
        *out = nullptr;
        H2B_REQUIRE(n_elems >= 1 && n_elems <= ((size_t)1 << 30), "poly_alloc: size out of range");
        h2b_poly* p = new h2b_poly();
        p->n = n_elems;
        p->device = ctx->device;
        cudaError_t e = cudaMalloc(&p->p, n_elems * 32);
        if (e != cudaSuccess) {
            delete p;
            throw StatusError{e == cudaErrorMemoryAllocation ? H2B_ERR_OOM : H2B_ERR_CUDA, std::string("poly_alloc: ") + cudaGetErrorString(e)};
        }
        H2B_CUDA(cudaMemsetAsync(p->p, 0, n_elems * 32, ctx->stream));
        *out = p;
    });
}
void h2b_poly_free(h2b_ctx* ctx, h2b_poly* poly) {
    if (!poly) return;
    if (ctx) {
        std::lock_guard<std::mutex> lock(ctx->mu);
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);
        if (poly->p) cudaFree(poly->p);
    } else if (poly->p) {
        cudaFree(poly->p);
    }
    delete poly;
}
void* h2b_poly_device_ptr(const h2b_poly* poly) { return poly ? poly->p : nullptr; }
size_t h2b_poly_len(const h2b_poly* poly) { return poly ? poly->n : 0; }
int h2b_poly_upload(h2b_ctx* ctx, h2b_poly* poly, size_t offset, const uint64_t* host, size_t n) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(poly && (host || n == 0), "poly_upload: null pointer");
        H2B_REQUIRE(offset <= poly->n && n <= poly->n - offset, "poly_upload: range outside the polynomial");
        if (n == 0) return;
        H2B_CUDA(cudaMemcpyAsync((char*)poly->p + offset * 32, host, n * 32, cudaMemcpyHostToDevice, ctx->stream));
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));  // the host buffer is the caller's again on return
    });
}
int h2b_poly_upload_async(h2b_ctx* ctx, h2b_poly* poly, size_t offset, const uint64_t* pinned_host, size_t n) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(poly && (pinned_host || n == 0), "poly_upload_async: null pointer");
        H2B_REQUIRE(offset <= poly->n && n <= poly->n - offset, "poly_upload_async: range outside the polynomial");
        if (n) H2B_CUDA(cudaMemcpyAsync((char*)poly->p + offset * 32, pinned_host, n * 32, cudaMemcpyHostToDevice, ctx->stream));
    });
}
int h2b_poly_copy_dev(h2b_ctx* ctx, void* d_dst, const void* d_src, size_t n) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_dst && d_src) || n == 0, "poly_copy: null pointer");
        if (n) H2B_CUDA(cudaMemcpyAsync(d_dst, d_src, n * 32, cudaMemcpyDeviceToDevice, ctx->stream));
    });
}
int h2b_poly_zero(h2b_ctx* ctx, h2b_poly* poly) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(poly, "poly_zero: null pointer");
        H2B_CUDA(cudaMemsetAsync(poly->p, 0, poly->n * 32, ctx->stream));
    });
}
int h2b_poly_download(h2b_ctx* ctx, const h2b_poly* poly, size_t offset, uint64_t* host, size_t n) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(poly && (host || n == 0), "poly_download: null pointer");
        H2B_REQUIRE(offset <= poly->n && n <= poly->n - offset, "poly_download: range outside the polynomial");
        if (n == 0) return;
        H2B_CUDA(cudaMemcpyAsync(host, (const char*)poly->p + offset * 32, n * 32, cudaMemcpyDeviceToHost, ctx->stream));
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    });
}

int h2b_permutation_product_dev(h2b_ctx* ctx, const void* const* d_columns, const void* const* d_sigma, size_t n_cols, size_t first_col,
                                const uint64_t beta[4], const uint64_t gamma[4], uint32_t k, uint32_t blinding_factors,
                                const void* d_start, void* d_z) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_columns && d_sigma && beta && gamma && d_z, "permutation_product: null pointer");
        permutation_product_run(ctx, d_columns, d_sigma, n_cols, first_col, beta, gamma, k, blinding_factors, d_start, d_z);
    });
}
int h2b_lookup_product_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, const void* d_permuted_input,
                           const void* d_permuted_table, const uint64_t beta[4], const uint64_t gamma[4], uint32_t k,
                           uint32_t blinding_factors, void* d_z) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_input && d_table && d_permuted_input && d_permuted_table && beta && gamma && d_z, "lookup_product: null pointer");
        lookup_product_run(ctx, d_input, d_table, d_permuted_input, d_permuted_table, beta, gamma, k, blinding_factors, d_z);
    });
}
int h2b_fr_mul_elementwise_dev(h2b_ctx* ctx, const void* d_a, const void* d_b, size_t n, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_a && d_b && d_out) || n == 0, "fr_mul_elementwise: null pointer");
        fr_mul_elementwise_run(ctx, d_a, d_b, n, d_out);
    });
}
int h2b_eval_polynomial_batch_dev(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* xs, size_t m, size_t n, uint64_t* out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_polys && xs && out) || m == 0, "eval_polynomial_batch: null pointer");
        if (m == 0) return;
        H2B_REQUIRE(m <= 4096, "eval_polynomial_batch: at most 4096 evaluations per call");
        char* d_out = (char*)ctx->get(WS_OUT, m * 32);
        for (size_t j = 0; j < m; j++) H2B_REQUIRE(d_polys[j] || n == 0, "eval_polynomial_batch: null polynomial");
        eval_polynomial_batch_run(ctx, d_polys, xs, m, n, d_out);
        uint64_t* bounce = (uint64_t*)ctx->get_pinned(2, m * 32 < 4096 ? 4096 : m * 32);
        H2B_CUDA(cudaMemcpyAsync(bounce, d_out, m * 32, cudaMemcpyDeviceToHost, ctx->stream));
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
        memcpy(out, bounce, m * 32);
    });
}

}  // extern "C"
