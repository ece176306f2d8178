// selectors.cu — the selector conflict matrix of halo2's keygen_vk (compress_selectors, DESIGN.md §4.13): for S selector columns
// of 0/1 Lagrange values, which pairs are active on a common row.  Two kernels:
//   k_sel_pack       one warp per 32 rows of one column: the values become one ballot word each (bit r = the row is 1); a value
//                    that is neither 0 nor the Montgomery 1 lowers the first-bad cell index c 2^k + r (atomicMin);
//   k_sel_conflicts  one CTA per (pair i <= j, range of 64-bit words): OR of bits_i & bits_j, written to both halves of the matrix.
// S^2 n / 64 word operations on bitsets of n / 8 bytes per column (1 MB at k = 23): the columns are read once, by the pack.
// The call synchronises and frees its scratch before it returns.
#include "h2b_internal.cuh"
#include "field.cuh"

namespace h2b {

namespace {
struct SelScratch {
    void* p = nullptr;
    explicit SelScratch(size_t bytes) { H2B_CUDA(cudaMalloc(&p, bytes ? bytes : 1)); }
    ~SelScratch() { cudaFree(p); }
};
size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
}  // namespace

// bits: S columns of W64 64-bit words (2 W64 ballot words), the padding words zeroed by the caller
__global__ void __launch_bounds__(256) k_sel_pack(const uint64_t* const* __restrict__ cols, u32 n, u32 W32, u32* __restrict__ bits, u32 stride32,
                                                  unsigned long long* __restrict__ bad) {
    const u32 c = blockIdx.y, lane = threadIdx.x & 31;
    const u32 w = blockIdx.x * 8 + (threadIdx.x >> 5);  // warp-uniform
    if (w >= W32) return;
    const u32 row = w * 32 + lane;
    bool one = false;
    if (row < n) {
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(cols[c] + 4 * (size_t)row);
        const ulonglong2 a = __ldg(p), b = __ldg(p + 1);
        one = a.x == 0xac96341c4ffffffbULL && a.y == 0x36fc76959f60cd29ULL && b.x == 0x666ea36f7879462eULL && b.y == 0x0e0a77c19a07df2fULL;
        const bool zero = (a.x | a.y | b.x | b.y) == 0;
        if (!zero && !one) atomicMin(bad, (unsigned long long)c * n + row);
    }
    const u32 word = __ballot_sync(0xffffffffu, one);
    if (lane == 0) bits[(size_t)c * stride32 + w] = word;
}

// conflicts[i S + j] = conflicts[j S + i] = 1 iff bits_i & bits_j has a set bit in this CTA's word range (i <= j; the diagonal: the
// column is active somewhere)
__global__ void __launch_bounds__(256) k_sel_conflicts(const unsigned long long* __restrict__ bits, u32 S, u32 W64, u32 per_block,
                                                       uint8_t* __restrict__ conflicts) {
    const u32 i = blockIdx.x / S, j = blockIdx.x % S;
    if (j < i) return;  // CTA-uniform
    const unsigned long long *a = bits + (size_t)i * W64, *b = bits + (size_t)j * W64;
    const u32 lo = blockIdx.y * per_block, hi = min(W64, lo + per_block);
    unsigned long long acc = 0;
    for (u32 w = lo + threadIdx.x; w < hi; w += blockDim.x) acc |= __ldg(a + w) & __ldg(b + w);
    if (__syncthreads_or(acc != 0) && threadIdx.x == 0) {
        conflicts[(size_t)i * S + j] = 1;
        conflicts[(size_t)j * S + i] = 1;
    }
}

void selector_conflicts_run(h2b_ctx* ctx, const void* const* d_cols, size_t S, uint32_t k, uint8_t* conflicts) {
    H2B_REQUIRE(k >= 1 && k <= 28, "selector_conflicts: k out of range (1..28)");
    H2B_REQUIRE(S >= 1 && S <= H2B_SELECTORS_MAX, "selector_conflicts: 1..4096 selector columns");
    for (size_t c = 0; c < S; c++) H2B_REQUIRE(d_cols[c], "selector_conflicts: null column");
    const u32 n = 1u << k, W32 = (n + 31) / 32, W64 = (W32 + 1) / 2;
    const size_t bits_bytes = al256(S * (size_t)W64 * 8), ptr_bytes = al256(S * 8), mat_bytes = al256(S * S);
    SelScratch scratch(bits_bytes + ptr_bytes + mat_bytes + 256);
    char* base = static_cast<char*>(scratch.p);
    u32* bits = reinterpret_cast<u32*>(base);
    const uint64_t** cols = reinterpret_cast<const uint64_t**>(base + bits_bytes);
    uint8_t* mat = reinterpret_cast<uint8_t*>(base + bits_bytes + ptr_bytes);
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(base + bits_bytes + ptr_bytes + mat_bytes);
    H2B_CUDA(cudaMemcpyAsync(cols, d_cols, S * 8, cudaMemcpyHostToDevice, ctx->stream));
    H2B_CUDA(cudaMemsetAsync(bits, 0, bits_bytes, ctx->stream));  // the odd ballot word of k <= 5
    H2B_CUDA(cudaMemsetAsync(mat, 0, S * S, ctx->stream));
    H2B_CUDA(cudaMemsetAsync(bad, 0xff, 8, ctx->stream));
    k_sel_pack<<<dim3((W32 + 7) / 8, (u32)S), 256, 0, ctx->stream>>>(cols, n, W32, bits, 2 * W64, bad);
    H2B_CUDA(cudaGetLastError());
    const u32 per_block = 4096, chunks = (W64 + per_block - 1) / per_block;
    k_sel_conflicts<<<dim3((u32)(S * S), chunks), 256, 0, ctx->stream>>>(reinterpret_cast<const unsigned long long*>(bits), (u32)S, W64, per_block,
                                                                         mat);
    H2B_CUDA(cudaGetLastError());
    unsigned long long* bounce = static_cast<unsigned long long*>(ctx->get_pinned(0, 4096));
    H2B_CUDA(cudaMemcpyAsync(bounce, bad, 8, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaMemcpyAsync(conflicts, mat, S * S, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    const unsigned long long first_bad = bounce[0];
    if (first_bad != ~0ULL)
        throw StatusError{H2B_ERR_ARG, "selector_conflicts: selector column " + std::to_string(first_bad >> k) + " holds a value other than 0 or 1 at row " +
                                           std::to_string(first_bad & (n - 1))};
}

}  // namespace h2b
