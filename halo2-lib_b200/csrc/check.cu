// check.cu — MockProver::verify for the constraint system halo2-base builds, on the device: which rows of a witness break
// a gate, a lookup or a copy constraint (include/h2b200.h, "constraint check").  Every check flags its failing cells (one
// byte per cell), and one report per checked item is built from the flags alone:
//     flags -> per-tile counts (2048 flags per tile) -> exclusive scan of the tile counts -> the rows of rank < max_report
// so the report (failure count, then the smallest failing rows in ascending order) is the same on every run; no atomic
// decides an order.
//   gate:    the h2b_graph interpreter of quotient.cu (graph.cuh) on Lagrange columns, rotation shift 0, one thread per row;
//   lookup:  the table's rows sorted by canonical value (lookup.cu's sort_column), then a binary search per input row;
//   sigma:   an entry v = delta^c' omega^r' is decoded by v^n = delta^(c' n) (omega^n = 1: k squarings, matched against
//            delta^(c n) for c < n_cols) and w = v delta^-c' = omega^r', found in an open-addressing table of the omega
//            powers (u32 row slots, full-value compare, so the answer does not depend on the insertion order);
//   copies:  value(c, r) against value(map(c, r)), one thread per cell;
//   equalities of a builder (MockProver, include/h2b200_mock.hpp): value(a) against value(b), value(cell) against its
//            constant, one thread per equality; the distinct constants counted as runs of the sorted column.
#include "h2b_internal.cuh"
#include "field.cuh"
#include "graph.cuh"
#include "keys.cuh"
#include "fr_domain_consts.inc"

namespace h2b {

static constexpr u32 RP_TILE = 2048;  // flags per tile of the reports: 256 threads x 8
static constexpr u32 EMPTY_SLOT = 0xffffffffu;

// ---------------------------------------------------------------------------------------------------------------- reports
__device__ __forceinline__ u32 tile_mask(const uint8_t* f, u32 n, u32 i0) {
    u32 m = 0;
#pragma unroll
    for (u32 j = 0; j < 8; j++)
        if (i0 + j < n && f[i0 + j]) m |= 1u << j;
    return m;
}

// counts[item][tile] = flags set in the tile
__global__ void __launch_bounds__(256) k_report_tiles(const uint8_t* __restrict__ flags, u32 n, u32 tiles, u32* __restrict__ counts) {
    __shared__ u32 wsum[8];
    const u32 t = threadIdx.x, tile = blockIdx.x, item = blockIdx.y;
    const u32 c = __popc(tile_mask(flags + (size_t)item * n, n, tile * RP_TILE + 8 * t));
    const u32 s = __reduce_add_sync(0xffffffffu, c);
    if ((t & 31) == 0) wsum[t >> 5] = s;
    __syncthreads();
    if (t == 0) {
        u32 tot = 0;
        for (int w = 0; w < 8; w++) tot += wsum[w];
        counts[(size_t)item * tiles + tile] = tot;
    }
}

// counts[item][*] -> exclusive prefixes in place; report word 0 = the item's failure count
__global__ void __launch_bounds__(1024) k_report_scan(u32* __restrict__ counts, u32 tiles, u32 report_words, uint64_t* __restrict__ reports) {
    __shared__ u32 wsum[32];
    const u32 t = threadIdx.x, lane = t & 31, warp = t >> 5, item = blockIdx.x;
    u32* c = counts + (size_t)item * tiles;
    u32 carry = 0;
    for (u32 j0 = 0; j0 < tiles; j0 += 1024) {
        const u32 j = j0 + t;
        const u32 v = j < tiles ? c[j] : 0;
        u32 inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (u32)d) inc += o;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        u32 before = 0, tot = 0;
        for (u32 w = 0; w < 32; w++) {
            before += w < warp ? wsum[w] : 0;
            tot += wsum[w];
        }
        if (j < tiles) c[j] = carry + before + inc - v;
        carry += tot;
        __syncthreads();
    }
    if (t == 0) reports[(size_t)item * report_words] = carry;
}

// the failing rows of rank < max_report: rank = failures in earlier tiles + failures earlier in this tile
__global__ void __launch_bounds__(256) k_report_rows(const uint8_t* __restrict__ flags, u32 n, u32 tiles, const u32* __restrict__ prefix,
                                                     u32 max_report, uint64_t* __restrict__ reports) {
    __shared__ u32 wsum[8];
    const u32 t = threadIdx.x, lane = t & 31, warp = t >> 5, tile = blockIdx.x, item = blockIdx.y;
    const u32 base = prefix[(size_t)item * tiles + tile];
    if (base >= max_report) return;  // the whole CTA: every row of this tile ranks too high
    const u32 i0 = tile * RP_TILE + 8 * t;
    u32 m = tile_mask(flags + (size_t)item * n, n, i0);
    const u32 c = __popc(m);
    u32 inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= (u32)d) inc += o;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    u32 rank = base + inc - c;
    for (u32 w = 0; w < warp; w++) rank += wsum[w];
    uint64_t* rep = reports + (size_t)item * (max_report + 1) + 1;
    while (m && rank < max_report) {
        const u32 j = __ffs(m) - 1;
        rep[rank++] = i0 + j;
        m &= m - 1;
    }
}

// m items of n flags each (item stride n bytes) -> m reports of max_report + 1 words, every word written
static void report_run(h2b_ctx* ctx, const uint8_t* d_flags, size_t m, u32 n, size_t max_report, void* d_reports, u32* counts) {
    const u32 tiles = ceil_div(n, RP_TILE);
    H2B_CUDA(cudaMemsetAsync(d_reports, 0, m * (max_report + 1) * 8, ctx->stream));
    H2B_LAUNCH(ctx, k_report_tiles, dim3(tiles, (unsigned)m), 256, 0, d_flags, n, tiles, counts);
    H2B_LAUNCH(ctx, k_report_scan, (unsigned)m, 1024, 0, counts, tiles, (u32)(max_report + 1), (uint64_t*)d_reports);
    H2B_LAUNCH(ctx, k_report_rows, dim3(tiles, (unsigned)m), 256, 0, d_flags, n, tiles, (const u32*)counts, (u32)max_report,
               (uint64_t*)d_reports);
}

// flag bytes for m items of n cells, then the tile counts of their reports (one workspace slot)
static uint8_t* flags_workspace(h2b_ctx* ctx, size_t m, u32 n, u32** counts) {
    const size_t fbytes = (m * n + 15) & ~(size_t)15;
    char* w = (char*)ctx->get(WS_CHECK_FLAGS, fbytes + m * ceil_div(n, RP_TILE) * 4);
    *counts = (u32*)(w + fbytes);
    return (uint8_t*)w;
}

static void check_common(uint32_t k, size_t max_report) {
    H2B_REQUIRE(k >= 1 && k <= 28, "check: k out of range (1..28)");
    H2B_REQUIRE(max_report >= 1 && max_report <= H2B_CHECK_MAX_REPORT, "check: max_report must be in 1..H2B_CHECK_MAX_REPORT");
}

// ------------------------------------------------------------------------------------------------------------------ gates
__global__ void __launch_bounds__(128) k_check_graph(GraphDev g, u32 k, u32 rows, uint8_t* __restrict__ flags) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows) return;
    Fr inter[H2B_GRAPH_MAX_CALCULATIONS];
    flags[idx] = graph_eval(g, idx, ((size_t)1 << k) - 1, 0, Fr::zero(), inter).is_zero() ? 0 : 1;
}

void check_graph_run(h2b_ctx* ctx, const h2b_graph* g, uint32_t k, size_t rows, size_t max_report, void* d_report) {
    check_common(k, max_report);
    H2B_REQUIRE(rows >= 1 && rows <= ((size_t)1 << k), "check_graph: rows must be in 1..2^k");
    const GraphDev gd = graph_upload(ctx, g);
    u32* counts;
    uint8_t* flags = flags_workspace(ctx, 1, (u32)rows, &counts);
    H2B_LAUNCH(ctx, k_check_graph, ceil_div(rows, 128), 128, 0, gd, k, (u32)rows, flags);
    report_run(ctx, flags, 1, (u32)rows, max_report, d_report, counts);
}

// ----------------------------------------------------------------------------------------------------------------- lookup
__global__ void __launch_bounds__(256) k_check_lookup(const uint64_t* __restrict__ input, const uint64_t* __restrict__ t_canon, u32 rows,
                                                      uint8_t* __restrict__ flags) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const Fr v = Fr::load_nc(input + 4 * (size_t)i).from_mont();
    Key256 key;
#pragma unroll
    for (int j = 0; j < 4; j++) key.l[j] = (uint64_t)v.l[2 * j] | ((uint64_t)v.l[2 * j + 1] << 32);
    flags[i] = sorted_contains(t_canon, rows, key) ? 0 : 1;
}

void check_lookup_run(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, size_t rows, size_t max_report, void* d_report) {
    check_common(k, max_report);
    H2B_REQUIRE(rows >= 1 && rows <= ((size_t)1 << k), "check_lookup: rows must be in 1..2^k");
    const u32 n = (u32)rows;
    const int sort_ctas = sort_column_ctas(ctx, n);
    const size_t scratch = sort_column_scratch(n, sort_ctas);
    // workspace: sort scratch | sorted table | its canonical values
    char* w = (char*)ctx->get(WS_SORT_TMP, scratch + 2 * (size_t)n * 32);
    uint64_t* t_sorted = (uint64_t*)(w + scratch);
    uint64_t* t_canon = t_sorted + 4 * (size_t)n;
    sort_column(ctx, (const uint64_t*)d_table, n, t_sorted, t_canon, w, sort_ctas);
    u32* counts;
    uint8_t* flags = flags_workspace(ctx, 1, n, &counts);
    H2B_LAUNCH(ctx, k_check_lookup, ceil_div(n, 256), 256, 0, (const uint64_t*)d_input, (const uint64_t*)t_canon, n, flags);
    report_run(ctx, flags, 1, n, max_report, d_report, counts);
}

// ------------------------------------------------------------------------------------------------------------ sigma decode
struct OmegaPow2 {
    uint64_t w[28][4];  // [j] = omega^(2^j) of the 2^k domain, j < k
};

__device__ __forceinline__ u32 fr_hash(const Fr& x, u32 mask) {
    const uint64_t lo = (uint64_t)x.l[0] | ((uint64_t)x.l[1] << 32);
    return (u32)((lo * 0x9e3779b97f4a7c15ull) >> 32) & mask;
}

// dn[c] = delta^(c n), dinv[c] = delta^-c for c < n_cols
__global__ void k_decode_delta(Fr delta, u32 k, u32 n_cols, uint64_t* __restrict__ dn, uint64_t* __restrict__ dinv) {
    const u32 c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_cols) return;
    Fr d_n = delta;
    for (u32 i = 0; i < k; i++) d_n = d_n.sqr();
    const Fr d_inv = delta.inv_bgcd();
    Fr a = Fr::one(), b = Fr::one();
    for (u32 j = 0; j < c; j++) {
        a = a * d_n;
        b = b * d_inv;
    }
    a.store(dn + 4 * (size_t)c);
    b.store(dinv + 4 * (size_t)c);
}

// pw[r] = omega^r, and row r entered into the open-addressing table (linear probing)
__global__ void __launch_bounds__(256) k_decode_omega(OmegaPow2 wp, u32 k, uint64_t* __restrict__ pw, u32* __restrict__ slots, u32 mask) {
    const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >> k) return;
    Fr x = Fr::one();
    for (u32 j = 0; j < k; j++)
        if ((r >> j) & 1) x = x * Fr::load(wp.w[j]);
    x.store(pw + 4 * (size_t)r);
    for (u32 h = fr_hash(x, mask);; h = (h + 1) & mask)
        if (atomicCAS(slots + h, EMPTY_SLOT, r) == EMPTY_SLOT) break;
}

struct DecodeDev {
    const uint64_t* const* sigma;
    const uint64_t* dn;
    const uint64_t* dinv;
    const uint64_t* pw;
    const u32* slots;
    u32 mask, n_cols, k;
};

// map[c][r] = c' << k | r' where sigma_c(r) = delta^c' omega^r'; a malformed entry is flagged and maps to its own cell
__global__ void __launch_bounds__(256) k_decode_sigma(DecodeDev d, u32* __restrict__ map, uint8_t* __restrict__ flags) {
    const u32 r = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y;
    if (r >> d.k) return;
    const size_t cell = ((size_t)c << d.k) + r;
    const Fr v = Fr::load_nc(d.sigma[c] + 4 * (size_t)r);
    Fr p = v;
    for (u32 i = 0; i < d.k; i++) p = p.sqr();
    u32 col = d.n_cols;
    for (u32 j = 0; j < d.n_cols; j++)
        if (p == Fr::load_nc(d.dn + 4 * (size_t)j)) {
            col = j;
            break;
        }
    u32 out = (c << d.k) | r;
    bool bad = true;
    if (col < d.n_cols) {
        const Fr w = v * Fr::load_nc(d.dinv + 4 * (size_t)col);
        for (u32 h = fr_hash(w, d.mask);; h = (h + 1) & d.mask) {
            const u32 s = __ldg(d.slots + h);
            if (s == EMPTY_SLOT) break;
            if (Fr::load_nc(d.pw + 4 * (size_t)s) == w) {
                out = (col << d.k) | s;
                bad = false;
                break;
            }
        }
    }
    map[cell] = out;
    flags[cell] = bad ? 1 : 0;
}

static void check_columns(const void* const* cols, size_t n_cols, uint32_t k, const char* what) {
    H2B_REQUIRE(n_cols >= 1 && n_cols < 65536, std::string(what) + ": n_cols must be in 1..65535");
    H2B_REQUIRE((size_t)k + ceil_log2(n_cols) <= 32, std::string(what) + ": k + ceil(log2 n_cols) > 32 (a map entry is 32 bits)");
    for (size_t i = 0; i < n_cols; i++) H2B_REQUIRE(cols[i], std::string(what) + ": null column");
}

// host array of device pointers -> device (workspace slot WS_MISC, staged from pageable memory before the call returns)
static const uint64_t* const* upload_pointers(h2b_ctx* ctx, const void* const* p, size_t m, size_t extra_bytes, char** extra) {
    const size_t pb = (8 * m + 255) & ~(size_t)255;
    char* d = (char*)ctx->get(WS_MISC, pb + extra_bytes);
    H2B_CUDA(cudaMemcpyAsync(d, p, 8 * m, cudaMemcpyHostToDevice, ctx->stream));
    *extra = d + pb;
    return (const uint64_t* const*)d;
}

void permutation_decode_run(h2b_ctx* ctx, const void* const* d_sigma, size_t n_cols, uint32_t k, void* d_map, size_t max_report,
                            void* d_reports) {
    check_common(k, max_report);
    check_columns(d_sigma, n_cols, k, "permutation_decode");
    const size_t n = (size_t)1 << k, cap = 2 * n;  // load factor 1/2
    char* dtab;
    DecodeDev d;
    d.sigma = upload_pointers(ctx, d_sigma, n_cols, 2 * 32 * n_cols, &dtab);
    d.dn = (const uint64_t*)dtab;
    d.dinv = d.dn + 4 * n_cols;
    char* t = (char*)ctx->get(WS_CHECK_TABLES, 32 * n + 4 * cap);
    d.pw = (const uint64_t*)t;
    d.slots = (const u32*)(t + 32 * n);
    d.mask = (u32)(cap - 1);
    d.n_cols = (u32)n_cols;
    d.k = k;
    Fr delta;
    memcpy(&delta, FR_DELTA_U64, sizeof(Fr));
    OmegaPow2 wp;
    for (uint32_t j = 0; j < k; j++) memcpy(wp.w[j], FR_OMEGA[k - j], 32);  // omega_k^(2^j) = omega_(k-j)
    H2B_CUDA(cudaMemsetAsync((void*)d.slots, 0xff, 4 * cap, ctx->stream));
    H2B_LAUNCH(ctx, k_decode_delta, ceil_div(n_cols, 64), 64, 0, delta, k, (u32)n_cols, (uint64_t*)d.dn, (uint64_t*)d.dinv);
    H2B_LAUNCH(ctx, k_decode_omega, ceil_div(n, 256), 256, 0, wp, k, (uint64_t*)d.pw, (u32*)d.slots, d.mask);
    u32* counts;
    uint8_t* flags = flags_workspace(ctx, n_cols, (u32)n, &counts);
    H2B_LAUNCH(ctx, k_decode_sigma, dim3(ceil_div(n, 256), (unsigned)n_cols), 256, 0, d, (u32*)d_map, flags);
    report_run(ctx, flags, n_cols, (u32)n, max_report, d_reports, counts);
}

// ----------------------------------------------------------------------------------------------------------------- copies
// a map entry naming a column >= n_cols counts as a failure (nothing is read through it)
__global__ void __launch_bounds__(256) k_check_copies(const uint64_t* const* __restrict__ cols, const u32* __restrict__ map, u32 n_cols, u32 k,
                                                      uint8_t* __restrict__ flags) {
    const u32 r = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y;
    if (r >> k) return;
    const size_t cell = ((size_t)c << k) + r;
    const u32 m = __ldg(map + cell), c2 = m >> k, r2 = m & ((1u << k) - 1);
    bool bad = true;
    if (c2 < n_cols) bad = !(Fr::load_nc(cols[c] + 4 * (size_t)r) - Fr::load_nc(cols[c2] + 4 * (size_t)r2)).is_zero();
    flags[cell] = bad ? 1 : 0;
}

void check_copies_run(h2b_ctx* ctx, const void* const* d_columns, const void* d_map, size_t n_cols, uint32_t k, size_t max_report,
                      void* d_reports) {
    check_common(k, max_report);
    check_columns(d_columns, n_cols, k, "check_copies");
    const size_t n = (size_t)1 << k;
    char* unused;
    const uint64_t* const* cols = upload_pointers(ctx, d_columns, n_cols, 0, &unused);
    u32* counts;
    uint8_t* flags = flags_workspace(ctx, n_cols, (u32)n, &counts);
    H2B_LAUNCH(ctx, k_check_copies, dim3(ceil_div(n, 256), (unsigned)n_cols), 256, 0, cols, (const u32*)d_map, (u32)n_cols, k, flags);
    report_run(ctx, flags, n_cols, (u32)n, max_report, d_reports, counts);
}

// ------------------------------------------------------------------------------------------ equalities of the builder
// halo2-base's copy manager as pairs of virtual-column cells: advice_equalities (a, b) and constant_equalities (c, i).  One
// thread per equality; an index >= N is not read, flags its equality and sets bit 0 of *status.
__global__ void __launch_bounds__(256) k_check_equalities(const uint64_t* __restrict__ cells, uint64_t N, const uint64_t* __restrict__ pairs,
                                                          u32 m, uint8_t* __restrict__ flags, u32* __restrict__ status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t a = __ldg(pairs + 2 * (size_t)i), b = __ldg(pairs + 2 * (size_t)i + 1);
    bool bad = true;
    if (a < N && b < N)
        bad = !(Fr::load_nc(cells + 4 * a) - Fr::load_nc(cells + 4 * b)).is_zero();
    else
        atomicOr(status, 1u);
    flags[i] = bad ? 1 : 0;
}

__global__ void __launch_bounds__(256) k_check_constants(const uint64_t* __restrict__ cells, uint64_t N, const uint64_t* __restrict__ consts,
                                                         const uint64_t* __restrict__ index, u32 m, uint8_t* __restrict__ flags,
                                                         u32* __restrict__ status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t a = __ldg(index + i);
    bool bad = true;
    if (a < N)
        bad = !(Fr::load_nc(cells + 4 * a) - Fr::load_nc(consts + 4 * (size_t)i)).is_zero();
    else
        atomicOr(status, 1u);
    flags[i] = bad ? 1 : 0;
}

// runs of equal values in a column of canonical values sorted ascending
__global__ void __launch_bounds__(256) k_count_runs(const uint64_t* __restrict__ canon, u32 m, u32* __restrict__ count) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    bool head = false;
    if (i < m) {
        head = i == 0;
        for (int j = 0; j < 4 && !head; j++) head = __ldg(canon + 4 * (size_t)i + j) != __ldg(canon + 4 * (size_t)i - 4 + j);
    }
    const u32 c = __popc(__ballot_sync(0xffffffffu, head));
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

static void check_pairs_common(size_t m, size_t max_report) {
    H2B_REQUIRE(max_report >= 1 && max_report <= H2B_CHECK_MAX_REPORT, "check: max_report must be in 1..H2B_CHECK_MAX_REPORT");
    H2B_REQUIRE(m < ((size_t)1 << 32), "check: at most 2^32 - 1 equalities per call");
}

void check_equalities_run(h2b_ctx* ctx, const void* d_cells, size_t N, const uint64_t* d_pairs, size_t m, size_t max_report, void* d_report,
                          uint32_t* d_status) {
    check_pairs_common(m, max_report);
    H2B_CUDA(cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    if (m == 0) {
        H2B_CUDA(cudaMemsetAsync(d_report, 0, (max_report + 1) * 8, ctx->stream));
        return;
    }
    u32* counts;
    uint8_t* flags = flags_workspace(ctx, 1, (u32)m, &counts);
    H2B_LAUNCH(ctx, k_check_equalities, ceil_div(m, 256), 256, 0, (const uint64_t*)d_cells, (uint64_t)N, d_pairs, (u32)m, flags, d_status);
    report_run(ctx, flags, 1, (u32)m, max_report, d_report, counts);
}

void check_constants_run(h2b_ctx* ctx, const void* d_cells, size_t N, const void* d_consts, const uint64_t* d_index, size_t m,
                         size_t max_report, void* d_report, uint32_t* d_status) {
    check_pairs_common(m, max_report);
    H2B_CUDA(cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    if (m == 0) {
        H2B_CUDA(cudaMemsetAsync(d_report, 0, (max_report + 1) * 8, ctx->stream));
        return;
    }
    u32* counts;
    uint8_t* flags = flags_workspace(ctx, 1, (u32)m, &counts);
    H2B_LAUNCH(ctx, k_check_constants, ceil_div(m, 256), 256, 0, (const uint64_t*)d_cells, (uint64_t)N, (const uint64_t*)d_consts, d_index,
               (u32)m, flags, d_status);
    report_run(ctx, flags, 1, (u32)m, max_report, d_report, counts);
}

void count_distinct_run(h2b_ctx* ctx, const void* d_values, size_t m, uint32_t* d_count) {
    H2B_REQUIRE(m < ((size_t)1 << 32), "count_distinct: at most 2^32 - 1 values");
    H2B_CUDA(cudaMemsetAsync(d_count, 0, 4, ctx->stream));
    if (m == 0) return;
    const u32 n = (u32)m;
    const int sort_ctas = sort_column_ctas(ctx, n);
    const size_t scratch = sort_column_scratch(n, sort_ctas);
    char* w = (char*)ctx->get(WS_SORT_TMP, scratch + 2 * (size_t)n * 32);
    uint64_t* sorted = (uint64_t*)(w + scratch);
    uint64_t* canon = sorted + 4 * (size_t)n;
    sort_column(ctx, (const uint64_t*)d_values, n, sorted, canon, w, sort_ctas);
    H2B_LAUNCH(ctx, k_count_runs, ceil_div(n, 256), 256, 0, (const uint64_t*)canon, n, d_count);
}

}  // namespace h2b
