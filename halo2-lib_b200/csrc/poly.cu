// poly.cu — opening arithmetic of the SHPLONK prover for sm_90a (SURVEY.md §8(f) rank 4):
//     eval_polynomial(poly, x)   = sum_i a_i x^i                      (halo2-axiom 0.5.3 arithmetic.rs)
//     kate_division(a, z)        = quotient of a(X) by (X - z)          (same file; the remainder a(z) is dropped)
//     linear combinations of polynomials                                (poly/kzg/multiopen/shplonk/prover.rs)
// None of these sources is vendored in the reference tree: the functions are restated from their definitions
// (outputs are mathematically unique), parity unpinned like the rest of L0.
//
// Both the evaluation and the division are the suffix recurrence  V(p) = a_p + x * V(p + 1),  V(n) = 0:
// a(x) = V(0) and q_{p-1} = V(p).  The recurrence is affine, so it is scanned in tiles: every CTA reduces a tile of
// 2048 coefficients to the value of the tile's polynomial at x, one CTA combines the tile values into the carry
// entering each tile from above, and a second pass replays the tile with its carry.  All kernels are HBM-bound:
// 32 B read per coefficient and pass, 32 B written per quotient coefficient.
#include "h2b_internal.cuh"
#include "field.cuh"

namespace h2b {

static constexpr int PD_TILE = 2048;  // 256 threads x 8 contiguous coefficients

// pw[j] = x^(2^j), j < 12 (x^8 and x^2048 are the chunk and tile weights)
__global__ void k_pow2_table(Fr x, uint64_t* __restrict__ pw) {
    if (threadIdx.x | blockIdx.x) return;
    for (int j = 0; j < 12; j++) {
        x.store(pw + 4 * j);
        x = x.sqr();
    }
}

// Suffix scan of an affine recurrence over the 256 threads of a CTA: on entry thread t holds c_t, the value of its
// chunk polynomial; all chunks span `w`-weighted equal lengths (w = x^len).  Returns D_t = c_t + w * D_{t+1}
// (D_256 = 0), i.e. the value at x of everything from the start of chunk t to the end of the CTA's range.
__device__ __forceinline__ Fr block_suffix_affine(Fr c, Fr w, Fr* sh /* 256 */) {
    const int t = threadIdx.x;
    c.store(sh + t);
    __syncthreads();
    for (int d = 1; d < 256; d <<= 1) {
        Fr o = Fr::zero();
        if (t + d < 256) o = Fr::load(sh + t + d);
        __syncthreads();
        if (t + d < 256) { c = c + w * o; c.store(sh + t); }
        __syncthreads();
        w = w.sqr();
    }
    return c;
}

__device__ __forceinline__ Fr chunk_value(const Fr v[8], const Fr& x) {  // Horner over 8 coefficients
    Fr r = v[7];
#pragma unroll
    for (int j = 6; j >= 0; j--) r = r * x + v[j];
    return r;
}

// tile_val[b] = sum_{i in tile b} a_i x^(i - tile start)
__global__ void __launch_bounds__(256) k_pd_tiles(const uint64_t* __restrict__ a, size_t n, const uint64_t* __restrict__ pw,
                                                  uint64_t* __restrict__ tile_val) {
    __shared__ Fr sh[256];
    const size_t base = (size_t)blockIdx.x * PD_TILE + (size_t)threadIdx.x * 8;
    Fr v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = (base + j < n) ? Fr::load_nc(a + 4 * (base + j)) : Fr::zero();
    const Fr x = Fr::load_nc(pw), x8 = Fr::load_nc(pw + 4 * 3);
    Fr d = block_suffix_affine(chunk_value(v, x), x8, sh);
    if (threadIdx.x == 0) d.store(tile_val + 4 * (size_t)blockIdx.x);
}

// carry[b] = V((b + 1) * TILE) = sum over the tiles above b; single CTA.  total = V(0) = a(x).
__device__ __forceinline__ void pd_scan_block(const uint64_t* __restrict__ tile_val, u32 ntiles, const uint64_t* __restrict__ pw,
                                              uint64_t* __restrict__ carry, uint64_t* __restrict__ total, Fr* sh /* 256 */) {
    const u32 per = (ntiles + 255) / 256;
    const u32 lo = min(threadIdx.x * per, ntiles), hi = min(lo + per, ntiles);
    const Fr xt = Fr::load_nc(pw + 4 * 11);  // x^2048
    Fr c = Fr::zero();
    for (u32 j = hi; j > lo; j--) c = c * xt + Fr::load_nc(tile_val + 4 * (size_t)(j - 1));
    // w = xt^per (uniform)
    Fr w = Fr::one(), sq = xt;
    for (u32 e = per; e; e >>= 1) {
        if (e & 1) w = w * sq;
        sq = sq.sqr();
    }
    Fr d = block_suffix_affine(c, w, sh);
    __syncthreads();
    d.store(sh + threadIdx.x);
    __syncthreads();
    Fr run = (threadIdx.x + 1 < 256) ? Fr::load(sh + threadIdx.x + 1) : Fr::zero();  // V(hi * TILE)
    for (u32 j = hi; j > lo; j--) {
        run.store(carry + 4 * (size_t)(j - 1));
        run = Fr::load_nc(tile_val + 4 * (size_t)(j - 1)) + xt * run;
    }
    if (threadIdx.x == 0 && total) d.store(total);
}
__global__ void __launch_bounds__(256) k_pd_scan(const uint64_t* __restrict__ tile_val, u32 ntiles, const uint64_t* __restrict__ pw,
                                                 uint64_t* __restrict__ carry, uint64_t* __restrict__ total) {
    __shared__ Fr sh[256];
    pd_scan_block(tile_val, ntiles, pw, carry, total, sh);
}

// q[i - 1] = V(i) for 1 <= i < n
__global__ void __launch_bounds__(256) k_pd_apply(const uint64_t* __restrict__ a, size_t n, const uint64_t* __restrict__ pw,
                                                  const uint64_t* __restrict__ carry, uint64_t* __restrict__ q) {
    __shared__ Fr sh[256];
    const size_t base = (size_t)blockIdx.x * PD_TILE + (size_t)threadIdx.x * 8;
    Fr v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = (base + j < n) ? Fr::load_nc(a + 4 * (base + j)) : Fr::zero();
    const Fr x = Fr::load_nc(pw), x8 = Fr::load_nc(pw + 4 * 3);
    Fr c = chunk_value(v, x);
    if (threadIdx.x == 255) c = c + x8 * Fr::load_nc(carry + 4 * (size_t)blockIdx.x);  // seed the scan with the tile's carry
    block_suffix_affine(c, x8, sh);
    // sh[t] = V(start of chunk t) after the scan's last store; the carry into chunk t is V(start of chunk t + 1)
    Fr run = (threadIdx.x == 255) ? Fr::load_nc(carry + 4 * (size_t)blockIdx.x) : Fr::load(sh + threadIdx.x + 1);
#pragma unroll
    for (int j = 7; j >= 0; j--) {
        run = v[j] + x * run;  // V(base + j)
        const size_t i = base + j;
        if (i >= 1 && i < n) run.store(q + 4 * (i - 1));
    }
}

static void pd_prepare(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t x[4], uint64_t** pw, uint64_t** tv, uint64_t** carry,
                       uint64_t** total, u32* ntiles) {
    *ntiles = (u32)((n + PD_TILE - 1) / PD_TILE);
    uint64_t* ws = (uint64_t*)ctx->get(WS_MISC2, 32 * (33 + 2 * (size_t)*ntiles));
    *pw = ws;
    *total = ws + 4 * 32;
    *tv = ws + 4 * 33;
    *carry = *tv + 4 * (size_t)*ntiles;
    Fr xx;
    memcpy(&xx, x, sizeof(Fr));
    H2B_LAUNCH(ctx, k_pow2_table, 1, 32, 0, xx, *pw);
    H2B_LAUNCH(ctx, k_pd_tiles, *ntiles, 256, 0, (const uint64_t*)d_a, n, *pw, *tv);
    H2B_LAUNCH(ctx, k_pd_scan, 1, 256, 0, *tv, *ntiles, *pw, *carry, *total);
}

// writes a(x) to d_out (device, 32 bytes)
void eval_polynomial_run(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t x[4], void* d_out) {
    if (n == 0) {
        H2B_CUDA(cudaMemsetAsync(d_out, 0, 32, ctx->stream));
        return;
    }
    uint64_t *pw, *tv, *carry, *total;
    u32 ntiles;
    pd_prepare(ctx, d_a, n, x, &pw, &tv, &carry, &total, &ntiles);
    H2B_CUDA(cudaMemcpyAsync(d_out, total, 32, cudaMemcpyDeviceToDevice, ctx->stream));
}

void kate_division_run(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t z[4], void* d_q) {
    H2B_REQUIRE(n >= 1, "kate_division: empty polynomial");
    if (n == 1) return;
    uint64_t *pw, *tv, *carry, *total;
    u32 ntiles;
    pd_prepare(ctx, d_a, n, z, &pw, &tv, &carry, &total, &ntiles);
    H2B_LAUNCH(ctx, k_pd_apply, ntiles, 256, 0, (const uint64_t*)d_a, n, pw, carry, (uint64_t*)d_q);
}

// ---------------------------------------------------------------- division by a vanishing polynomial of m <= 4 points
// (a - r) / Z_T = sum_j w_j (a - a(z_j)) / (X - z_j),  Z_T = prod_j (X - z_j),  w_j = 1 / prod_{k != j} (z_j - z_k):
// the quotient of a by Z_T is a weighted sum of m kate_division quotients, i.e. of m independent suffix recurrences
// V_j(p) = a_p + z_j V_j(p + 1).  The passes of kate_division run for all m points at once: each CTA reads its tile of a
// once and carries m values; the apply pass writes the weighted sum once.
struct DivPoints {
    Fr z[H2B_KATE_MULTI_MAX], w[H2B_KATE_MULTI_MAX];
};
// pw[j] = the 12 powers z_j^(2^i) (as k_pow2_table), one thread per point
__global__ void k_pdm_pow2(DivPoints p, u32 m, uint64_t* __restrict__ pw) {
    if (threadIdx.x >= m) return;
    Fr x = p.z[threadIdx.x];
    for (int i = 0; i < 12; i++) {
        x.store(pw + 48 * threadIdx.x + 4 * i);
        x = x.sqr();
    }
}
// tile_val[j][b] as k_pd_tiles for every point
template <int M>
__global__ void __launch_bounds__(256) k_pdm_tiles(const uint64_t* __restrict__ a, size_t n, u32 ntiles, const uint64_t* __restrict__ pw,
                                                   uint64_t* __restrict__ tile_val) {
    __shared__ Fr sh[256];
    const size_t base = (size_t)blockIdx.x * PD_TILE + (size_t)threadIdx.x * 8;
    Fr v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = (base + j < n) ? Fr::load_nc(a + 4 * (base + j)) : Fr::zero();
#pragma unroll 1
    for (int j = 0; j < M; j++) {
        const Fr x = Fr::load_nc(pw + 48 * j), x8 = Fr::load_nc(pw + 48 * j + 4 * 3);
        Fr d = block_suffix_affine(chunk_value(v, x), x8, sh);
        if (threadIdx.x == 0) d.store(tile_val + 4 * ((size_t)j * ntiles + blockIdx.x));
        __syncthreads();  // the next point's scan rewrites sh
    }
}
// carry[j][b] as k_pd_scan, one CTA per point
__global__ void __launch_bounds__(256) k_pdm_scan(const uint64_t* __restrict__ tile_val, u32 ntiles, const uint64_t* __restrict__ pw,
                                                  uint64_t* __restrict__ carry) {
    __shared__ Fr sh[256];
    const size_t j = blockIdx.x;
    pd_scan_block(tile_val + 4 * j * ntiles, ntiles, pw + 48 * j, carry + 4 * j * ntiles, nullptr, sh);
}
// q[i - 1] = sum_j w_j V_j(i) for 1 <= i < n
template <int M>
__global__ void __launch_bounds__(256) k_pdm_apply(const uint64_t* __restrict__ a, size_t n, u32 ntiles, const uint64_t* __restrict__ pw,
                                                   const uint64_t* __restrict__ carry, DivPoints p, uint64_t* __restrict__ q) {
    __shared__ Fr sh[256];
    const size_t base = (size_t)blockIdx.x * PD_TILE + (size_t)threadIdx.x * 8;
    Fr v[8], acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        v[j] = (base + j < n) ? Fr::load_nc(a + 4 * (base + j)) : Fr::zero();
        acc[j] = Fr::zero();
    }
#pragma unroll 1
    for (int j = 0; j < M; j++) {
        const Fr x = Fr::load_nc(pw + 48 * j), x8 = Fr::load_nc(pw + 48 * j + 4 * 3);
        const Fr cin = Fr::load_nc(carry + 4 * ((size_t)j * ntiles + blockIdx.x));
        Fr c = chunk_value(v, x);
        if (threadIdx.x == 255) c = c + x8 * cin;
        block_suffix_affine(c, x8, sh);
        Fr run = (threadIdx.x == 255) ? cin : Fr::load(sh + threadIdx.x + 1);
        __syncthreads();  // every thread has read sh before the next point's scan rewrites it
        const Fr w = p.w[j];
#pragma unroll
        for (int t = 7; t >= 0; t--) {
            run = v[t] + x * run;
            acc[t] = acc[t] + w * run;
        }
    }
#pragma unroll
    for (int t = 0; t < 8; t++) {
        const size_t i = base + t;
        if (i >= 1 && i < n) acc[t].store(q + 4 * (i - 1));
    }
}

template <int M>
static void kate_division_multi_launch(h2b_ctx* ctx, const uint64_t* a, size_t n, u32 ntiles, uint64_t* pw, uint64_t* tv, uint64_t* carry,
                                       const DivPoints& p, uint64_t* q) {
    H2B_LAUNCH(ctx, k_pdm_tiles<M>, ntiles, 256, 0, a, n, ntiles, pw, tv);
    H2B_LAUNCH(ctx, k_pdm_scan, M, 256, 0, tv, ntiles, pw, carry);
    H2B_LAUNCH(ctx, k_pdm_apply<M>, ntiles, 256, 0, a, n, ntiles, pw, carry, p, q);
}

void kate_division_multi_run(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t* points, size_t m, const uint64_t* weights, void* d_q) {
    H2B_REQUIRE(n >= 1, "kate_division_multi: empty polynomial");
    H2B_REQUIRE(m >= 1 && m <= H2B_KATE_MULTI_MAX, "kate_division_multi: 1..4 points");
    if (n == 1) return;
    DivPoints p;
    memset(&p, 0, sizeof(p));
    memcpy(p.z, points, 32 * m);
    memcpy(p.w, weights, 32 * m);
    const u32 ntiles = (u32)((n + PD_TILE - 1) / PD_TILE);
    uint64_t* pw = (uint64_t*)ctx->get(WS_MISC2, 32 * (12 * m + 2 * m * (size_t)ntiles));
    uint64_t* tv = pw + 48 * m;
    uint64_t* carry = tv + 4 * m * (size_t)ntiles;
    H2B_LAUNCH(ctx, k_pdm_pow2, 1, 32, 0, p, (u32)m, pw);
    const uint64_t* a = (const uint64_t*)d_a;
    uint64_t* q = (uint64_t*)d_q;
    switch (m) {
        case 1: kate_division_multi_launch<1>(ctx, a, n, ntiles, pw, tv, carry, p, q); break;
        case 2: kate_division_multi_launch<2>(ctx, a, n, ntiles, pw, tv, carry, p, q); break;
        case 3: kate_division_multi_launch<3>(ctx, a, n, ntiles, pw, tv, carry, p, q); break;
        default: kate_division_multi_launch<4>(ctx, a, n, ntiles, pw, tv, carry, p, q); break;
    }
}

// ---------------------------------------------------------------- batched evaluation
// m (polynomial, point) pairs in three launches: blockIdx.y selects the pair.  The evaluations create_proof writes after
// the challenge x are ~25 Horner sums over 2^k coefficients each; one at a time they are latency-bound (three small
// launches per evaluation).
struct EvalBatch {
    const uint64_t* const* polys;  // device array of m pointers
    const uint64_t* xs;            // device, m x 4
};
__global__ void k_pow2_table_batch(EvalBatch b, uint64_t* __restrict__ pw /* m x 12 x 4 */) {
    if (threadIdx.x) return;
    Fr x = Fr::load(b.xs + 4 * (size_t)blockIdx.x);
    uint64_t* o = pw + 48 * (size_t)blockIdx.x;
    for (int j = 0; j < 12; j++) {
        x.store(o + 4 * j);
        x = x.sqr();
    }
}
__global__ void __launch_bounds__(256) k_pd_tiles_batch(EvalBatch b, size_t n, u32 ntiles, const uint64_t* __restrict__ pw,
                                                        uint64_t* __restrict__ tile_val /* m x ntiles x 4 */) {
    __shared__ Fr sh[256];
    const uint64_t* a = b.polys[blockIdx.y];
    const uint64_t* mypw = pw + 48 * (size_t)blockIdx.y;
    const size_t base = (size_t)blockIdx.x * PD_TILE + (size_t)threadIdx.x * 8;
    Fr v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = (base + j < n) ? Fr::load_nc(a + 4 * (base + j)) : Fr::zero();
    const Fr x = Fr::load_nc(mypw), x8 = Fr::load_nc(mypw + 4 * 3);
    Fr d = block_suffix_affine(chunk_value(v, x), x8, sh);
    if (threadIdx.x == 0) d.store(tile_val + 4 * ((size_t)blockIdx.y * ntiles + blockIdx.x));
}
// one CTA per pair: Horner over the tile values with x^2048 (ntiles is at most a few thousand)
__global__ void __launch_bounds__(256) k_pd_scan_batch(const uint64_t* __restrict__ tile_val, u32 ntiles, const uint64_t* __restrict__ pw,
                                                       uint64_t* __restrict__ out /* m x 4 */) {
    __shared__ Fr sh[256];
    const uint64_t* tv = tile_val + 4 * (size_t)blockIdx.x * ntiles;
    const uint64_t* mypw = pw + 48 * (size_t)blockIdx.x;
    const u32 per = (ntiles + 255) / 256;
    const u32 lo = min(threadIdx.x * per, ntiles), hi = min(lo + per, ntiles);
    const Fr xt = Fr::load_nc(mypw + 4 * 11);  // x^2048
    Fr c = Fr::zero();
    for (u32 j = hi; j > lo; j--) c = c * xt + Fr::load_nc(tv + 4 * (size_t)(j - 1));
    Fr w = Fr::one(), sq = xt;
    for (u32 e = per; e; e >>= 1) {
        if (e & 1) w = w * sq;
        sq = sq.sqr();
    }
    Fr d = block_suffix_affine(c, w, sh);
    if (threadIdx.x == 0) d.store(out + 4 * (size_t)blockIdx.x);
}

// d_polys: host array of m device pointers; xs: host, m x 4; d_out: device, m x 4
void eval_polynomial_batch_run(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* xs, size_t m, size_t n, void* d_out) {
    if (m == 0) return;
    if (n == 0) {
        H2B_CUDA(cudaMemsetAsync(d_out, 0, m * 32, ctx->stream));
        return;
    }
    const u32 ntiles = (u32)((n + PD_TILE - 1) / PD_TILE);
    // staging block: [pointers m x 8 | points m x 32], then device scratch: pow tables m x 12 x 32, tile values m x ntiles x 32
    const size_t head = ((m * 8 + 31) & ~(size_t)31), in_bytes = head + m * 32;
    char* h_in = (char*)ctx->get_pinned(1, in_bytes < 4096 ? 4096 : in_bytes);
    memcpy(h_in, d_polys, m * 8);
    memcpy(h_in + head, xs, m * 32);
    char* ws = (char*)ctx->get(WS_MISC2, in_bytes + m * 12 * 32 + (size_t)m * ntiles * 32 + 64);
    H2B_CUDA(cudaMemcpyAsync(ws, h_in, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    EvalBatch b{(const uint64_t* const*)ws, (const uint64_t*)(ws + head)};
    uint64_t* pw = (uint64_t*)(ws + ((in_bytes + 31) & ~(size_t)31));
    uint64_t* tv = pw + 48 * m;
    H2B_LAUNCH(ctx, k_pow2_table_batch, (unsigned)m, 32, 0, b, pw);
    H2B_LAUNCH(ctx, k_pd_tiles_batch, dim3(ntiles, (unsigned)m), 256, 0, b, n, ntiles, pw, tv);
    H2B_LAUNCH(ctx, k_pd_scan_batch, (unsigned)m, 256, 0, tv, ntiles, pw, (uint64_t*)d_out);
}

// ---------------------------------------------------------------- linear combination
struct LincombArgs {
    const uint64_t* polys[32];
    Fr scalars[32];
    int m;
};
__global__ void __launch_bounds__(256) k_poly_lincomb(const LincombArgs* __restrict__ args, size_t n, uint64_t* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int m = args->m;
    Fr acc = Fr::load(args->polys[0] + 4 * i) * args->scalars[0];
#pragma unroll 1
    for (int j = 1; j < m; j++) acc = acc + Fr::load(args->polys[j] + 4 * i) * args->scalars[j];
    acc.store(out + 4 * i);
}

void poly_lincomb_run(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* scalars, size_t m, size_t n, void* d_out) {
    H2B_REQUIRE(m >= 1 && m <= 32, "poly_lincomb: 1..32 polynomials per call");
    if (n == 0) return;
    LincombArgs host;
    memset(&host, 0, sizeof(host));
    for (size_t j = 0; j < m; j++) {
        H2B_REQUIRE(d_polys[j], "poly_lincomb: null polynomial");
        host.polys[j] = (const uint64_t*)d_polys[j];
        memcpy(&host.scalars[j], scalars + 4 * j, 32);
    }
    host.m = (int)m;
    void* d_args = ctx->get(WS_MISC, sizeof(LincombArgs));
    H2B_CUDA(cudaMemcpyAsync(d_args, &host, sizeof(host), cudaMemcpyHostToDevice, ctx->stream));
    H2B_LAUNCH(ctx, k_poly_lincomb, ceil_div(n, 256), 256, 0, (const LincombArgs*)d_args, n, (uint64_t*)d_out);
}

}  // namespace h2b
