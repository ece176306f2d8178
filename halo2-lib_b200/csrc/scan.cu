// scan.cu — Fr batch inversion and grand-product (prefix product) columns for sm_90a.
//
// These are the primitives behind the permutation / lookup grand products of create_proof (SURVEY.md §3.3 step 4,
// §8(f) rank 2; halo2-axiom 0.5.3 `plonk/permutation/prover.rs`, `plonk/lookup/prover.rs`, ff 0.13 `BatchInvert`):
//     denominators  d_i <- d_i^-1  (zeros stay zero, as `BatchInvert::batch_invert` skips them)
//     z[0] = start, z[i] = z[i-1] * f[i-1]                      (`z.push(z[row - 1] * modified_values[row - 1])`)
// and of the prover's `batch_invert_assigned` for `Assigned::Rational` witness cells (h2b_eval_rational).
#include "h2b_internal.cuh"
#include "field.cuh"

namespace h2b {

// ---------------------------------------------------------------- batch inversion
// One Fermat inversion per CTA of 256 threads x E elements (thread t owns elements base + e*256 + t, coalesced):
//   1. every thread multiplies its non-zero elements;  2. block-wide exclusive prefix / suffix products of the thread
//   totals;  3. thread 0 inverts the CTA total (binary extended Euclid, Fp::inv_bgcd: the only long dependency chain,
//   which the other resident CTAs cover);  4. thread t starts from u = total^-1 * (product of the threads after t)
//   and walks its elements backwards: a_i^-1 = u * (everything before i), u *= a_i.
// 4 products per element plus the scans; the per-thread inversion this replaces cost ~47 products per element.
__device__ __forceinline__ Fr block_exclusive_prefix_product(Fr v, Fr* sh /* 256 */, Fr* total);

__device__ __forceinline__ Fr block_exclusive_suffix_product(Fr v, Fr* sh /* 256 */) {
    const int t = threadIdx.x;
    __syncthreads();
    v.store(sh + t);
    __syncthreads();
    for (int d = 1; d < 256; d <<= 1) {
        Fr o = Fr::one();
        if (t + d < 256) o = Fr::load(sh + t + d);
        __syncthreads();
        if (t + d < 256) { v = v * o; v.store(sh + t); }
        __syncthreads();
    }
    Fr ex = (t == 255) ? Fr::one() : Fr::load(sh + t + 1);
    __syncthreads();
    return ex;
}

__global__ void __launch_bounds__(256) k_batch_invert(uint64_t* __restrict__ a, uint64_t* __restrict__ scratch, size_t n, int E) {
    __shared__ Fr sh[256];
    __shared__ Fr sh_inv;
    const size_t base = (size_t)blockIdx.x * 256 * E + threadIdx.x;
    Fr mine = Fr::one();
    for (int e = 0; e < E; e++) {
        const size_t i = base + (size_t)e * 256;
        if (i >= n) break;
        Fr v = Fr::load(a + 4 * i);
        if (!v.is_zero()) mine = mine * v;
    }
    Fr total;
    const Fr before = block_exclusive_prefix_product(mine, sh, &total);
    const Fr after = block_exclusive_suffix_product(mine, sh);
    if (threadIdx.x == 0) sh_inv = total.inv_bgcd();  // one lane: the product-free inversion has the shorter chain
    // forward again: running product of everything before element i (threads before me, then my earlier elements)
    Fr run = before;
    for (int e = 0; e < E; e++) {
        const size_t i = base + (size_t)e * 256;
        if (i >= n) break;
        Fr v = Fr::load(a + 4 * i);
        run.store(scratch + 4 * i);
        if (!v.is_zero()) run = run * v;
    }
    __syncthreads();
    Fr u = sh_inv * after;  // inverse of the product of everything up to and including my last element
    for (int e = E - 1; e >= 0; e--) {
        const size_t i = base + (size_t)e * 256;
        if (i >= n) continue;
        Fr v = Fr::load(a + 4 * i);
        if (v.is_zero()) continue;
        (u * Fr::load(scratch + 4 * i)).store(a + 4 * i);
        u = u * v;
    }
}

// out[i] = num[i] * den[i]  (after den has been inverted in place)
__global__ void __launch_bounds__(256) k_mul_elementwise(const uint64_t* __restrict__ x, const uint64_t* __restrict__ y, size_t n,
                                                         uint64_t* __restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    (Fr::load_nc(x + 4 * i) * Fr::load_nc(y + 4 * i)).store(out + 4 * i);
}

void batch_invert_run(h2b_ctx* ctx, void* d_a, size_t n) {
    if (n == 0) return;
    // one wave of CTAs (4 of these fit an SM at 64 registers per thread), so that every CTA's inversion chain runs
    // concurrently: a second wave would add a full ~165 us chain; at most 16 elements per thread
    const size_t slots = (size_t)256 * 4 * ctx->sm_count;
    int E = (int)((n + slots - 1) / slots);
    if (E < 2) E = 2;
    if (E > 16) E = 16;
    uint64_t* scratch = (uint64_t*)ctx->get(WS_MISC2, n * 32);
    H2B_LAUNCH(ctx, k_batch_invert, ceil_div(n, (size_t)256 * E), 256, 0, (uint64_t*)d_a, scratch, n, E);
}

// ---------------------------------------------------------------- grand product
// Tile = 2048 elements per CTA (256 threads x 8 contiguous).  k_gp_tiles: product of every tile.  k_gp_scan: single
// CTA, exclusive prefix products of the tile totals times `start`.  k_gp_apply: exclusive prefix inside the tile.
static constexpr int GP_TILE = 2048;

__device__ __forceinline__ Fr block_exclusive_prefix_product(Fr v, Fr* sh /* 256 */, Fr* total) {
    // Hillis-Steele inclusive scan under multiplication over 256 threads, returns the exclusive prefix of thread t
    const int t = threadIdx.x;
    v.store(sh + t);
    __syncthreads();
    for (int d = 1; d < 256; d <<= 1) {
        Fr o = Fr::one();
        if (t >= d) o = Fr::load(sh + t - d);
        __syncthreads();
        if (t >= d) { v = o * v; v.store(sh + t); }
        __syncthreads();
    }
    if (total) *total = Fr::load(sh + 255);
    Fr ex = (t == 0) ? Fr::one() : Fr::load(sh + t - 1);
    __syncthreads();
    return ex;
}

__global__ void __launch_bounds__(256) k_gp_tiles(const uint64_t* __restrict__ f, size_t n_f, uint64_t* __restrict__ tile_prod) {
    __shared__ Fr sh[256];
    const size_t base = (size_t)blockIdx.x * GP_TILE + (size_t)threadIdx.x * 8;
    Fr p = Fr::one();
    for (int j = 0; j < 8; j++)
        if (base + j < n_f) p = p * Fr::load_nc(f + 4 * (base + j));
    Fr total;
    block_exclusive_prefix_product(p, sh, &total);
    if (threadIdx.x == 0) total.store(tile_prod + 4 * (size_t)blockIdx.x);
}
// exclusive prefix over the tile totals, seeded with `start`: tile_base[j] = start * prod_{j' < j} tile_prod[j']
__global__ void __launch_bounds__(256) k_gp_scan(const uint64_t* __restrict__ tile_prod, u32 ntiles, Fr start,
                                                 uint64_t* __restrict__ tile_base, const uint64_t* __restrict__ d_start) {
    __shared__ Fr sh[256];
    if (d_start) start = Fr::load(d_start);
    const u32 per = (ntiles + 255) / 256;
    const u32 lo = min(threadIdx.x * per, ntiles), hi = min(lo + per, ntiles);
    Fr p = Fr::one();
    for (u32 j = lo; j < hi; j++) p = p * Fr::load_nc(tile_prod + 4 * (size_t)j);
    Fr run = start * block_exclusive_prefix_product(p, sh, nullptr);
    for (u32 j = lo; j < hi; j++) {
        run.store(tile_base + 4 * (size_t)j);
        run = run * Fr::load_nc(tile_prod + 4 * (size_t)j);
    }
}
// z[i] = tile_base[tile] * prod_{tile start <= j < i} f[j]   for i < n_z
__global__ void __launch_bounds__(256) k_gp_apply(const uint64_t* __restrict__ f, size_t n_f, const uint64_t* __restrict__ tile_base,
                                                  uint64_t* __restrict__ z, size_t n_z) {
    __shared__ Fr sh[256];
    const size_t base = (size_t)blockIdx.x * GP_TILE + (size_t)threadIdx.x * 8;
    Fr v[8], p = Fr::one();
    for (int j = 0; j < 8; j++) {
        v[j] = (base + j < n_f) ? Fr::load_nc(f + 4 * (base + j)) : Fr::one();
        p = p * v[j];
    }
    Fr run = Fr::load_nc(tile_base + 4 * (size_t)blockIdx.x) * block_exclusive_prefix_product(p, sh, nullptr);
    for (int j = 0; j < 8; j++) {
        if (base + j < n_z) run.store(z + 4 * (base + j));
        run = run * v[j];
    }
}

// z[0] = start, z[i] = z[i-1] * f[i-1], i < n  (f[n-1] is not used, as in halo2)
void grand_product_run(h2b_ctx* ctx, const void* d_f, const uint64_t start[4], size_t n, void* d_z, const void* d_start) {
    if (n == 0) return;
    const size_t n_f = n - 1;
    const u32 ntiles = (u32)((n + GP_TILE - 1) / GP_TILE);
    uint64_t* tp = (uint64_t*)ctx->get(WS_MISC2, (size_t)ntiles * 2 * 32);
    uint64_t* tb = tp + 4 * (size_t)ntiles;
    Fr s;
    memcpy(&s, start, sizeof(Fr));
    H2B_LAUNCH(ctx, k_gp_tiles, ntiles, 256, 0, (const uint64_t*)d_f, n_f, tp);
    H2B_LAUNCH(ctx, k_gp_scan, 1, 256, 0, tp, ntiles, s, tb, (const uint64_t*)d_start);
    H2B_LAUNCH(ctx, k_gp_apply, ntiles, 256, 0, (const uint64_t*)d_f, n_f, tb, (uint64_t*)d_z, n);
}

// Assigned::Rational cells: out = num * den^-1 (den = 0 -> 0); den is copied, inverted as a batch, multiplied
void eval_rational_batched_run(h2b_ctx* ctx, const void* d_num, const void* d_den, size_t n, void* d_out) {
    if (n == 0) return;
    void* tmp = ctx->get(WS_MISC, n * 32);
    H2B_CUDA(cudaMemcpyAsync(tmp, d_den, n * 32, cudaMemcpyDeviceToDevice, ctx->stream));
    batch_invert_run(ctx, tmp, n);
    H2B_LAUNCH(ctx, k_mul_elementwise, ceil_div(n, 256), 256, 0, (const uint64_t*)d_num, (const uint64_t*)tmp, n, (uint64_t*)d_out);
}

}  // namespace h2b
