// lookup.cu — the lookup argument's permuted columns for sm_90a (SURVEY.md §8(f) rank 2):
// halo2-axiom 0.5.3 `plonk/lookup/prover.rs::permute_expression_pair` (not vendored; restated from the upstream
// algorithm).  Given the compressed input column A and table column S over the usable rows u = n - (blinding + 1):
//     A' = A sorted by Fr's `Ord` (integer order of the canonical value);
//     S'[row] = A'[row]                         where A' starts a new run (first occurrence of the value),
//     S'[row] = a left-over table value         elsewhere: the sorted table minus the first instance of every distinct
//                                               input value, in ascending order.
// WHICH repeated row receives which left-over value is not determined by the protocol, and the forks differ:
//   * the sorted-table walk of PSE halo2 >= 2023 and the forks derived from it — which is what halo2-axiom 0.5.3 is
//     recalled to carry (not vendored, cannot be confirmed here: DESIGN.md §2) — fills the unfilled rows FRONT TO BACK
//     (two cursors over the sorted table and the distinct inputs): the default here;
//   * zcash halo2 iterates a BTreeMap of left-over counts and pops the repeated rows from the BACK
//     (`repeated_input_rows.pop()`): h2b_ctx_set_option("lookup.leftover_order", 1).
// Either column satisfies the argument; only proof BYTES depend on the choice.
// An input value that is not in the table is `Error::ConstraintSystemFailure` (H2B_ERR_UNSATISFIED here).
//
// Sorting 254-bit keys: a stable LSD radix sort of a ROW PERMUTATION over the 32 bytes of the canonical values, written
// here (no library sort): ONE cooperative launch per column (k_radix_sort) loops over the byte positions with grid-wide
// barriers; k_canon leaves the OR of (value XOR first value) over the column, so every CTA skips the byte positions that
// are constant over the column without asking the host — range-check columns carry < 2^lookup_bits values, two passes are
// the common case.  A pass: per-CTA digit histogram of its contiguous segment -> bin-major table -> row scans -> stable
// scatter (rank inside a 256-element tile by __match_any_sync + per-warp counters).  Everything else is flag / scan /
// scatter work (own two-launch scan), HBM-bound on 32-byte records.  The verdict ("an input value is missing") stays in
// device memory for the _async entry point; only the synchronous entry points read it back.
#include <algorithm>
#include <cooperative_groups.h>

#include "h2b_internal.cuh"
#include "field.cuh"
#include "keys.cuh"

namespace cg = cooperative_groups;

namespace h2b {

// canonical (non-Montgomery) values, the identity permutation, and diff[0..8) |= value XOR first value (a byte position
// whose bits are all zero there is constant over the column: its sort pass is the identity)
__global__ void __launch_bounds__(256) k_canon(const uint64_t* __restrict__ src, u32 n, uint64_t* __restrict__ canon, u32* __restrict__ idx,
                                               u32* __restrict__ diff) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 mine[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (i < n) {
        Fr v = Fr::load_nc(src + 4 * (size_t)i).from_mont();
        v.store(canon + 4 * (size_t)i);
        idx[i] = i;
        Fr first = Fr::load_nc(src).from_mont();
#pragma unroll
        for (int l = 0; l < 8; l++) mine[l] = v.l[l] ^ first.l[l];
    }
#pragma unroll
    for (int l = 0; l < 8; l++) {
        const u32 m = __reduce_or_sync(0xffffffffu, mine[l]);
        if ((threadIdx.x & 31) == 0 && m) atomicOr(diff + l, m);
    }
}

// Stable LSD radix sort of the permutation idx_a by the canonical keys, 8 bits per pass, one cooperative launch.
// table: 256 x gridDim.x counters (bin-major), totals: 256.  Result in idx_a or idx_b: *which = 0 / 1.
static constexpr int RS_T = 256;
__global__ void __launch_bounds__(RS_T) k_radix_sort(const uint64_t* __restrict__ canon, u32 n, u32* __restrict__ idx_a, u32* __restrict__ idx_b,
                                                     const u32* __restrict__ diff, u32* __restrict__ table, u32* __restrict__ totals,
                                                     u32* __restrict__ which) {
    cg::grid_group grid = cg::this_grid();
    __shared__ u32 hist[256];
    __shared__ u32 base[256];
    __shared__ u32 wcnt[RS_T / 32][256];
    const u32 t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const u32 G = gridDim.x, cta = blockIdx.x;
    // contiguous segment of this CTA, whole tiles of RS_T elements (the order inside the segment is the input order)
    const u32 tiles = (n + RS_T - 1) / RS_T;
    const u32 t_lo = (u32)((uint64_t)tiles * cta / G), t_hi = (u32)((uint64_t)tiles * (cta + 1) / G);
    const u32 seg_lo = t_lo * RS_T, seg_hi = min(n, t_hi * RS_T);
    const uint8_t* keys = reinterpret_cast<const uint8_t*>(canon);
    u32* src = idx_a;
    u32* dst = idx_b;
    u32 flips = 0;
    for (int pos = 0; pos < 32; pos++) {
        if (((__ldg(diff + (pos >> 2)) >> (8 * (pos & 3))) & 0xffu) == 0) continue;  // constant byte: identity pass
        // ---- histogram of the segment
        hist[t] = 0;
        __syncthreads();
        for (u32 i = seg_lo + t; i < seg_hi; i += RS_T) atomicAdd(&hist[keys[32 * (size_t)src[i] + pos]], 1u);
        __syncthreads();
        table[(size_t)t * G + cta] = hist[t];
        grid.sync();
        // ---- row scans: CTA b (and b + G, ...) turns row b into exclusive prefixes and leaves the row total
        for (u32 b = cta; b < 256; b += G) {
            u32* row = table + (size_t)b * G;
            u32 carry = 0;
            for (u32 j0 = 0; j0 < G; j0 += RS_T) {
                const u32 j = j0 + t;
                const u32 v = j < G ? row[j] : 0;
                u32 inc = v;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
                    if (lane >= (u32)d) inc += o;
                }
                if (lane == 31) hist[warp] = inc;
                __syncthreads();
                u32 wb = 0;
                for (u32 w = 0; w < warp; w++) wb += hist[w];
                u32 tot = 0;
                for (u32 w = 0; w < RS_T / 32; w++) tot += hist[w];
                if (j < G) row[j] = carry + wb + inc - v;
                carry += tot;
                __syncthreads();
            }
            if (t == 0) totals[b] = carry;
        }
        grid.sync();
        // ---- base[bin] = entries of smaller bins + entries of this bin in earlier CTAs
        {
            const u32 v = totals[t];
            u32 inc = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= (u32)d) inc += o;
            }
            if (lane == 31) hist[warp] = inc;
            __syncthreads();
            u32 wb = 0;
            for (u32 w = 0; w < warp; w++) wb += hist[w];
            base[t] = wb + inc - v + table[(size_t)t * G + cta];
            __syncthreads();
        }
        // ---- stable scatter, tile by tile
        for (u32 i0 = seg_lo; i0 < seg_hi; i0 += RS_T) {
            const u32 i = i0 + t;
            const bool live = i < seg_hi;
            u32 id = 0, dg = 0;
            if (live) { id = src[i]; dg = keys[32 * (size_t)id + pos]; }
            for (u32 e = t; e < (RS_T / 32) * 256; e += RS_T) (&wcnt[0][0])[e] = 0;
            __syncthreads();
            const unsigned act = __ballot_sync(0xffffffffu, live);
            u32 rank_in_warp = 0;
            if (live) {
                const unsigned peers = __match_any_sync(act, dg);
                rank_in_warp = __popc(peers & ((1u << lane) - 1));
                if (rank_in_warp == 0) wcnt[warp][dg] = __popc(peers);
            }
            __syncthreads();
            if (live) {
                u32 before = 0;
                for (u32 w = 0; w < warp; w++) before += wcnt[w][dg];
                dst[base[dg] + before + rank_in_warp] = id;
            }
            __syncthreads();
            u32 add = 0;
            for (u32 w = 0; w < RS_T / 32; w++) add += wcnt[w][t];
            base[t] += add;
            __syncthreads();
        }
        grid.sync();
        u32* tmp = src; src = dst; dst = tmp;
        flips++;
    }
    if (cta == 0 && t == 0) *which = flips & 1u;
}
__global__ void __launch_bounds__(256) k_gather_rows(const uint64_t* __restrict__ src, const uint64_t* __restrict__ canon,
                                                     const u32* __restrict__ idx_a, const u32* __restrict__ idx_b, const u32* __restrict__ which,
                                                     u32 n, uint64_t* __restrict__ out, uint64_t* __restrict__ out_canon) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t j = (__ldg(which) ? idx_b : idx_a)[i];
    Fr::load_nc(src + 4 * j).store(out + 4 * (size_t)i);
    Fr::load_nc(canon + 4 * j).store(out_canon + 4 * (size_t)i);
}

// rep[i] = 1 where A'[i] repeats A'[i-1]; left[j] = 1 where table value j is NOT consumed by a first occurrence;
// *missing |= 1 when a first occurrence is absent from the table
__global__ void __launch_bounds__(256) k_lookup_flags(const uint64_t* __restrict__ a_canon, const uint64_t* __restrict__ t_canon, u32 n,
                                                      u32* __restrict__ rep, u32* __restrict__ left, u32* __restrict__ missing) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Key256 a = key_load(a_canon, i), t = key_load(t_canon, i);
    const bool a_first = i == 0 || key_cmp(key_load(a_canon, i - 1), a) != 0;
    const bool t_first = i == 0 || key_cmp(key_load(t_canon, i - 1), t) != 0;
    rep[i] = a_first ? 0u : 1u;
    if (a_first && !sorted_contains(t_canon, n, a)) atomicOr(missing, 1u);
    left[i] = (t_first && sorted_contains(a_canon, n, t)) ? 0u : 1u;
}
// rep_rows[rank] = row for the repeated rows, ascending
__global__ void __launch_bounds__(256) k_lookup_rep_rows(const u32* __restrict__ rep, const u32* __restrict__ rep_pos, u32 n, u32* __restrict__ rep_rows) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && rep[i]) rep_rows[rep_pos[i]] = i;
}
// S' : first occurrences copy A'; left-over number q (ascending) goes to the repeated row of rank q (front to back), or of
// rank R-1-q when `backward` (the zcash order)
__global__ void __launch_bounds__(256) k_lookup_fill(const uint64_t* __restrict__ a_sorted, const uint64_t* __restrict__ t_sorted,
                                                     const u32* __restrict__ rep, const u32* __restrict__ rep_pos, const u32* __restrict__ left,
                                                     const u32* __restrict__ left_pos, const u32* __restrict__ rep_rows, u32 n,
                                                     uint64_t* __restrict__ s_out, u32* __restrict__ missing, int backward) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 n_rep = rep_pos[n - 1] + rep[n - 1], n_left = left_pos[n - 1] + left[n - 1];
    if (n_rep != n_left) {  // cannot happen when every input value is in the table
        if (i == 0) atomicOr(missing, 2u);
        return;
    }
    if (!rep[i]) Fr::load_nc(a_sorted + 4 * (size_t)i).store(s_out + 4 * (size_t)i);
    if (left[i]) Fr::load_nc(t_sorted + 4 * (size_t)i).store(s_out + 4 * (size_t)rep_rows[backward ? n_rep - 1 - left_pos[i] : left_pos[i]]);
}

// Exclusive scans of the two flag arrays at once (tile = 2048 flags per CTA): tiles -> tile sums -> add the preceding sums.
static constexpr int XS_TILE = 2048;
__global__ void __launch_bounds__(256) k_xscan_tiles(const u32* __restrict__ fa, const u32* __restrict__ fb, u32 n, u32* __restrict__ pa,
                                                     u32* __restrict__ pb, uint2* __restrict__ tile_sums) {
    __shared__ uint2 wsum[8];
    const u32 t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const u32 i0 = blockIdx.x * XS_TILE + t * 8;
    u32 va[8], vb[8], sa = 0, sb = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        va[j] = i0 + j < n ? fa[i0 + j] : 0;
        vb[j] = i0 + j < n ? fb[i0 + j] : 0;
        sa += va[j];
        sb += vb[j];
    }
    u32 ia = sa, ib = sb;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 oa = __shfl_up_sync(0xffffffffu, ia, d), ob = __shfl_up_sync(0xffffffffu, ib, d);
        if (lane >= (u32)d) { ia += oa; ib += ob; }
    }
    if (lane == 31) wsum[warp] = make_uint2(ia, ib);
    __syncthreads();
    u32 wa = 0, wb = 0;
    for (u32 w = 0; w < warp; w++) { wa += wsum[w].x; wb += wsum[w].y; }
    u32 ra = wa + ia - sa, rb = wb + ib - sb;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (i0 + j < n) { pa[i0 + j] = ra; pb[i0 + j] = rb; }
        ra += va[j];
        rb += vb[j];
    }
    if (t == 255) tile_sums[blockIdx.x] = make_uint2(ra, rb);
}
__global__ void __launch_bounds__(256) k_xscan_apply(u32 n, const uint2* __restrict__ tile_sums, u32* __restrict__ pa, u32* __restrict__ pb) {
    __shared__ uint2 red[256];
    const u32 t = threadIdx.x;
    u32 sa = 0, sb = 0;
    for (u32 j = t; j < blockIdx.x; j += 256) { sa += tile_sums[j].x; sb += tile_sums[j].y; }
    red[t] = make_uint2(sa, sb);
    __syncthreads();
    for (int d = 128; d >= 1; d >>= 1) {
        if (t < (u32)d) { red[t].x += red[t + d].x; red[t].y += red[t + d].y; }
        __syncthreads();
    }
    const u32 aa = red[0].x, ab = red[0].y, base = blockIdx.x * XS_TILE;
    if (aa == 0 && ab == 0) return;
    for (u32 e = t; e < XS_TILE; e += 256)
        if (base + e < n) { pa[base + e] += aa; pb[base + e] += ab; }
}

// cooperative grid of the sort: every CTA resident, no more CTAs than tiles
int sort_column_ctas(h2b_ctx* ctx, u32 n) {
    int per_sm = 0;
    H2B_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_radix_sort, RS_T, 0));
    H2B_REQUIRE(per_sm >= 1, "sort_column: the sort kernel does not fit on an SM");
    int sort_ctas = ctx->sm_count * (per_sm < 4 ? per_sm : 4);
    const int tiles = (int)((n + RS_T - 1) / RS_T);
    if (sort_ctas > tiles) sort_ctas = tiles;
    return sort_ctas;
}
size_t sort_column_scratch(u32 n, int sort_ctas) {
    return ((size_t)n * (32 + 4 + 4) + (256 * (size_t)sort_ctas + 256 + 16) * 4 + 255) & ~(size_t)255;
}

// sorts one column: out = src sorted by canonical value, out_canon = the canonical values in that order
void sort_column(h2b_ctx* ctx, const uint64_t* d_src, u32 n, uint64_t* d_out, uint64_t* d_out_canon, char* scratch, int sort_ctas) {
    // scratch: canon (32 n) | idx_a (4 n) | idx_b (4 n) | table (256 x CTAs) | totals (256) | diff (8) | which (1)
    uint64_t* canon = (uint64_t*)scratch;
    u32* idx_a = (u32*)(canon + 4 * (size_t)n);
    u32* idx_b = idx_a + n;
    u32* table = idx_b + n;
    u32* totals = table + 256 * (size_t)sort_ctas;
    u32* diff = totals + 256;
    u32* which = diff + 8;
    H2B_CUDA(cudaMemsetAsync(diff, 0, 9 * 4, ctx->stream));
    H2B_LAUNCH(ctx, k_canon, ceil_div(n, 256), 256, 0, d_src, n, canon, idx_a, diff);
    const uint64_t* c_canon = canon;
    const u32* c_diff = diff;
    void* args[] = {(void*)&c_canon, (void*)&n, (void*)&idx_a, (void*)&idx_b, (void*)&c_diff, (void*)&table, (void*)&totals, (void*)&which};
    H2B_CUDA(cudaLaunchCooperativeKernel((const void*)k_radix_sort, dim3((unsigned)sort_ctas), dim3(RS_T), args, 0, ctx->stream));
    ctx->launches++;
    H2B_LAUNCH(ctx, k_gather_rows, ceil_div(n, 256), 256, 0, d_src, c_canon, (const u32*)idx_a, (const u32*)idx_b, (const u32*)which, n, d_out,
               d_out_canon);
}

// ---------------------------------------------------------------------- the same sort and scan on integer keys (keygen.cu)
// idx = init (or the identity) and diff[0..8) |= key XOR first key: the byte positions k_radix_sort has to pass over
__global__ void __launch_bounds__(256) k_key_init(const uint64_t* __restrict__ keys, u32 n, const u32* __restrict__ init, u32* __restrict__ idx,
                                                  u32* __restrict__ diff) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 mine[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (i < n) {
        idx[i] = init ? init[i] : i;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint64_t x = __ldg(keys + 4 * (size_t)i + j) ^ __ldg(keys + j);
            mine[2 * j] = (u32)x;
            mine[2 * j + 1] = (u32)(x >> 32);
        }
    }
#pragma unroll
    for (int l = 0; l < 8; l++) {
        const u32 m = __reduce_or_sync(0xffffffffu, mine[l]);
        if ((threadIdx.x & 31) == 0 && m) atomicOr(diff + l, m);
    }
}
__global__ void __launch_bounds__(256) k_pick_perm(const u32* __restrict__ idx_a, const u32* __restrict__ idx_b, const u32* __restrict__ which, u32 n,
                                                   u32* __restrict__ perm) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) perm[i] = (__ldg(which) ? idx_b : idx_a)[i];
}

size_t sort_keys_scratch(u32 n, int sort_ctas) {
    return ((size_t)n * 8 + (256 * (size_t)sort_ctas + 256 + 16) * 4 + 255) & ~(size_t)255;
}

void sort_keys(h2b_ctx* ctx, const uint64_t* d_keys, u32 n, const u32* d_init, u32* d_perm, char* scratch, int sort_ctas) {
    if (n == 0) return;
    // scratch: idx_a (4 n) | idx_b (4 n) | table (256 x CTAs) | totals (256) | diff (8) | which (1)
    u32* idx_a = (u32*)scratch;
    u32* idx_b = idx_a + n;
    u32* table = idx_b + n;
    u32* totals = table + 256 * (size_t)sort_ctas;
    u32* diff = totals + 256;
    u32* which = diff + 8;
    H2B_CUDA(cudaMemsetAsync(diff, 0, 9 * 4, ctx->stream));
    H2B_LAUNCH(ctx, k_key_init, ceil_div(n, 256), 256, 0, d_keys, n, d_init, idx_a, diff);
    const u32* c_diff = diff;
    void* args[] = {(void*)&d_keys, (void*)&n, (void*)&idx_a, (void*)&idx_b, (void*)&c_diff, (void*)&table, (void*)&totals, (void*)&which};
    H2B_CUDA(cudaLaunchCooperativeKernel((const void*)k_radix_sort, dim3((unsigned)sort_ctas), dim3(RS_T), args, 0, ctx->stream));
    ctx->launches++;
    H2B_LAUNCH(ctx, k_pick_perm, ceil_div(n, 256), 256, 0, (const u32*)idx_a, (const u32*)idx_b, (const u32*)which, n, d_perm);
}

size_t exclusive_scan_scratch(u32 n) { return ((size_t)n * 4 + (size_t)ceil_div(n, XS_TILE) * 8 + 255) & ~(size_t)255; }

void exclusive_scan(h2b_ctx* ctx, const u32* d_in, u32 n, u32* d_out, char* scratch) {
    if (n == 0) return;
    const u32 ntiles = ceil_div(n, XS_TILE);
    u32* unused = (u32*)scratch;  // the second scan of the pair runs over the same flags
    uint2* tile_sums = (uint2*)(scratch + (((size_t)n * 4 + 7) & ~(size_t)7));
    H2B_LAUNCH(ctx, k_xscan_tiles, ntiles, 256, 0, d_in, d_in, n, d_out, unused, tile_sums);
    H2B_LAUNCH(ctx, k_xscan_apply, ntiles, 256, 0, n, (const uint2*)tile_sums, d_out, unused);
}

// Enqueues the whole permutation; the verdict word (bit 0: an input value is missing from the table, bit 1: counts
// disagree) is left at the returned device address, zero when the argument is satisfiable.
u32* permute_expression_pair_enqueue(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                     void* d_permuted_input, void* d_permuted_table) {
    H2B_REQUIRE(k <= 28, "permute_expression_pair: k out of range");
    const size_t rows = (size_t)1 << k;
    H2B_REQUIRE((size_t)blinding_factors + 1 < rows, "permute_expression_pair: no usable rows");
    const u32 n = (u32)(rows - (blinding_factors + 1));
    const int sort_ctas = sort_column_ctas(ctx, n);
    const u32 ntiles = (n + XS_TILE - 1) / XS_TILE;
    const size_t sort_scratch = sort_column_scratch(n, sort_ctas);
    // workspace: sort scratch | a_canon | t_sorted | t_canon | rep, rep_pos, left, left_pos, rep_rows | tile sums | missing
    const size_t total = sort_scratch + 3 * (size_t)n * 32 + 5 * (size_t)n * 4 + (size_t)ntiles * 8 + 256;
    char* w = (char*)ctx->get(WS_SORT_TMP, total);
    char* scratch = w;
    uint64_t* a_canon = (uint64_t*)(scratch + sort_scratch);
    uint64_t* t_sorted = a_canon + 4 * (size_t)n;
    uint64_t* t_canon = t_sorted + 4 * (size_t)n;
    u32* rep = (u32*)(t_canon + 4 * (size_t)n);
    u32 *rep_pos = rep + n, *left = rep_pos + n, *left_pos = left + n, *rep_rows = left_pos + n;
    uint2* tile_sums = (uint2*)(rep_rows + n + (n & 1));
    u32* missing = (u32*)(tile_sums + ntiles);
    H2B_CUDA(cudaMemsetAsync(missing, 0, 4, ctx->stream));
    sort_column(ctx, (const uint64_t*)d_input, n, (uint64_t*)d_permuted_input, a_canon, scratch, sort_ctas);
    sort_column(ctx, (const uint64_t*)d_table, n, t_sorted, t_canon, scratch, sort_ctas);
    H2B_LAUNCH(ctx, k_lookup_flags, ceil_div(n, 256), 256, 0, a_canon, t_canon, n, rep, left, missing);
    H2B_LAUNCH(ctx, k_xscan_tiles, ntiles, 256, 0, (const u32*)rep, (const u32*)left, n, rep_pos, left_pos, tile_sums);
    H2B_LAUNCH(ctx, k_xscan_apply, ntiles, 256, 0, n, (const uint2*)tile_sums, rep_pos, left_pos);
    H2B_LAUNCH(ctx, k_lookup_rep_rows, ceil_div(n, 256), 256, 0, rep, rep_pos, n, rep_rows);
    H2B_LAUNCH(ctx, k_lookup_fill, ceil_div(n, 256), 256, 0, (const uint64_t*)d_permuted_input, t_sorted, rep, rep_pos, left, left_pos, rep_rows, n,
               (uint64_t*)d_permuted_table, missing, ctx->opt_lookup_backward);
    return missing;
}

// returns true when some input value is missing from the table (one device-to-host read of the verdict word)
bool permute_expression_pair_run(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                 void* d_permuted_input, void* d_permuted_table) {
    const u32* missing = permute_expression_pair_enqueue(ctx, d_input, d_table, k, blinding_factors, d_permuted_input, d_permuted_table);
    u32* bounce = (u32*)ctx->get_pinned(0, 4096);
    H2B_CUDA(cudaMemcpyAsync(bounce, missing, 4, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    return bounce[0] != 0;
}

}  // namespace h2b
