// assign.cu — column-wise witness assignment for sm_90a.
//
// Replaces the per-cell loop of `assign_witnesses`
// (halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312; each cell goes through
// raw_assign_advice, utils/halo2.rs:20-27, into the prover's WitnessCollection) and the lookup-column copy
// of LookupAnyManager::assign_raw (halo2-base/src/virtual_region/lookups.rs:130-155).
//
// Closed form of the walk (SURVEY.md Appendix A.2): with V the concatenation of ctx.advice over threads,
// b_0..b_{m-1} the pinned break points and s_0 = 0, s_{c+1} = s_c + b_c, column c holds V[s_c + r] for
// 0 <= r <= b_c (the cell at the break is duplicated into row 0 of column c+1); the walk stops breaking as
// soon as fewer than b_c + 1 cells remain.  The kernels are pure 32-byte gathers: 64 B of traffic per cell.
#include "h2b_internal.cuh"
#include "field.cuh"

namespace h2b {

struct ColSpan {
    uint64_t start;  // s_c
    uint64_t len;    // cells in column c
};

__global__ void __launch_bounds__(256) k_assign_columns(const uint4* __restrict__ vcol, const ColSpan* __restrict__ spans,
                                                        u32 rows_log, u32 ncols, uint4* __restrict__ cols) {
    // one thread per 16-byte half cell: a warp moves 512 contiguous bytes
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = ((size_t)ncols << rows_log) * 2;
    if (g >= total) return;
    size_t cell = g >> 1;
    u32 half = (u32)(g & 1);
    u32 c = (u32)(cell >> rows_log);
    size_t r = cell & (((size_t)1 << rows_log) - 1);
    ColSpan sp = spans[c];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < sp.len) v = __ldg(vcol + 2 * (sp.start + r) + half);
    cols[g] = v;
}

struct ColSpans64 {
    ColSpan s[64];
};
// same gather with the spans passed by value (no staging copy, no host synchronisation): up to 64 columns
__global__ void __launch_bounds__(256) k_assign_columns_v(const uint4* __restrict__ vcol, ColSpans64 spans, u32 rows_log, u32 ncols,
                                                          uint4* __restrict__ cols) {
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = ((size_t)ncols << rows_log) * 2;
    if (g >= total) return;
    size_t cell = g >> 1;
    u32 half = (u32)(g & 1);
    u32 c = (u32)(cell >> rows_log);
    size_t r = cell & (((size_t)1 << rows_log) - 1);
    const ColSpan sp = spans.s[c];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < sp.len) v = __ldg(vcol + 2 * (sp.start + r) + half);
    cols[g] = v;
}

// `Assigned<Fr>` staging records (72 bytes: tag, numerator, denominator; halo2-base/src/lib.rs:157-188 re-exports the
// prover crate's Assigned::{Zero, Trivial(F), Rational(F, F)}): split into a numerator and a denominator array.
// tag 0 -> (0, 1), 1 -> (num, 1), 2 -> (num, den).  stats[0] counts the Rational cells, stats[1] the invalid tags.
__global__ void __launch_bounds__(256) k_assigned_split(const uint64_t* __restrict__ recs, size_t N, uint64_t* __restrict__ num,
                                                        uint64_t* __restrict__ den, u32* __restrict__ stats) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const uint64_t* r = recs + 9 * i;
    const uint64_t tag = __ldg(r);
    Fr nu = Fr::zero(), de = Fr::one();
    if (tag == 1 || tag == 2) {
        uint64_t w[4];
#pragma unroll
        for (int j = 0; j < 4; j++) w[j] = __ldg(r + 1 + j);
#pragma unroll
        for (int j = 0; j < 4; j++) { nu.l[2 * j] = (u32)w[j]; nu.l[2 * j + 1] = (u32)(w[j] >> 32); }
    }
    if (tag == 2) {
        uint64_t w[4];
#pragma unroll
        for (int j = 0; j < 4; j++) w[j] = __ldg(r + 5 + j);
#pragma unroll
        for (int j = 0; j < 4; j++) { de.l[2 * j] = (u32)w[j]; de.l[2 * j + 1] = (u32)(w[j] >> 32); }
        atomicAdd(stats, 1u);
    }
    if (tag > 2) atomicAdd(stats + 1, 1u);
    nu.store(num + 4 * i);
    de.store(den + 4 * i);
}

__global__ void __launch_bounds__(256) k_assign_lookups(const uint4* __restrict__ vals, size_t N, u32 rows_log, u32 L,
                                                        uint4* __restrict__ cols) {
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = ((size_t)L << rows_log) * 2;
    if (g >= total) return;
    size_t cell = g >> 1;
    u32 half = (u32)(g & 1);
    u32 c = (u32)(cell >> rows_log);
    size_t r = cell & (((size_t)1 << rows_log) - 1);
    size_t j = r * L + c;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (j < N) v = __ldg(vals + 2 * j + half);
    cols[g] = v;
}

// halo2-base form of the witness: lookup cell j = values[index[j]] (the copy LookupAnyManager::assign_raw makes), laid out
// as k_assign_lookups lays out the values.  An index >= N yields zero and sets bit 0 of *status.
__global__ void __launch_bounds__(256) k_assign_lookups_indexed(const uint4* __restrict__ vals, size_t N, const uint64_t* __restrict__ index,
                                                                size_t n_lookup, u32 rows_log, u32 L, uint4* __restrict__ cols,
                                                                u32* __restrict__ status) {
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = ((size_t)L << rows_log) * 2;
    if (g >= total) return;
    size_t cell = g >> 1;
    u32 half = (u32)(g & 1);
    u32 c = (u32)(cell >> rows_log);
    size_t r = cell & (((size_t)1 << rows_log) - 1);
    size_t j = r * L + c;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (j < n_lookup) {
        const uint64_t idx = __ldg(index + j);
        if (idx < N)
            v = __ldg(vals + 2 * idx + half);
        else if (half == 0)
            atomicOr(status, 1u);
    }
    cols[g] = v;
}

// Assigned::Rational(n, d) cells of the halo2-base form: values[index[i]] holds n, den_inv[i] = d^-1 (0 for d = 0).  Each
// thread checks its own entry: index[i] < N (else bit 0 of *status) and index[i] > index[i-1] (else bit 1).  A valid entry
// is the only writer of its cell, because the valid indices strictly increase.
__global__ void __launch_bounds__(256) k_apply_rational(uint64_t* __restrict__ values, size_t N, const uint64_t* __restrict__ index,
                                                        const uint64_t* __restrict__ den_inv, size_t R, u32* __restrict__ status) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    const uint64_t idx = __ldg(index + i);
    u32 bad = idx < N ? 0u : 1u;
    if (i > 0 && idx <= __ldg(index + i - 1)) bad |= 2u;
    if (bad) {
        atomicOr(status, bad);
        return;
    }
    (Fr::load(values + 4 * idx) * Fr::load_nc(den_inv + 4 * i)).store(values + 4 * idx);
}

// the spans of the ncols columns the walk fills: column c holds V[s_c .. s_c + len_c); columns the walk does not reach are empty
static std::vector<ColSpan> column_spans(size_t N, const uint64_t* break_points, size_t nbp, size_t rows, size_t ncols) {
    std::vector<ColSpan> spans(ncols, ColSpan{0, 0});
    size_t s = 0, c = 0, bpi = 0;
    size_t rem = N;
    while (rem > 0) {
        if (c >= ncols)
            throw StatusError{H2B_ERR_LAYOUT, "assign_witnesses: break points walk past the last advice column (single_phase.rs:304)"};
        // The walk compares row_offset with the break point only for cells it assigns in its main step; the
        // duplicate written at row 0 of a new column is not compared, so in columns c > 0 a break point of 0
        // can never fire (and, never being consumed, disables all later ones).
        const bool can_break = bpi < nbp && rem > break_points[bpi] && (c == 0 || break_points[bpi] >= 1);
        if (can_break) {
            size_t b = (size_t)break_points[bpi++];
            if (b + 1 > rows) throw StatusError{H2B_ERR_LAYOUT, "assign_witnesses: break point beyond the 2^k rows of a column"};
            spans[c] = ColSpan{s, b + 1};
            s += b;
            rem -= b;  // the duplicated cell + the rest
            c++;
            if (c >= ncols)
                throw StatusError{H2B_ERR_LAYOUT, "assign_witnesses: break points walk past the last advice column (single_phase.rs:304)"};
        } else {
            if (rem > rows) throw StatusError{H2B_ERR_LAYOUT, "assign_witnesses: column overflows 2^k rows"};
            spans[c] = ColSpan{s, rem};
            rem = 0;
        }
    }
    return spans;
}

void assign_columns_run(h2b_ctx* ctx, const void* d_vcol, size_t N, const uint64_t* break_points, size_t nbp,
                        uint32_t k, size_t ncols, void* d_cols) {
    H2B_REQUIRE(k <= 28, "assign: k out of range");
    const size_t rows = (size_t)1 << k;
    if (ncols == 0) {
        // single_phase.rs:279-286: "Trying to assign threads in a phase with no columns"
        if (N != 0) throw StatusError{H2B_ERR_LAYOUT, "assign_witnesses: cells present but the phase has no advice columns"};
        return;
    }
    const std::vector<ColSpan> spans = column_spans(N, break_points, nbp, rows, ncols);
    size_t total = ncols * rows * 2;
    if (ncols <= 64) {  // the usual case: spans travel as a kernel argument, the call stays asynchronous
        ColSpans64 sv;
        memset(&sv, 0, sizeof(sv));
        for (size_t i = 0; i < ncols; i++) sv.s[i] = spans[i];
        H2B_LAUNCH(ctx, k_assign_columns_v, ceil_div(total, 256), 256, 0, (const uint4*)d_vcol, sv, k, (u32)ncols, (uint4*)d_cols);
        return;
    }
    ColSpan* d_spans = (ColSpan*)ctx->get(WS_MISC, ncols * sizeof(ColSpan));
    ColSpan* h_spans = (ColSpan*)ctx->get_pinned(1, ncols * sizeof(ColSpan));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));  // > 64 columns: the pinned staging block may still be in flight
    memcpy(h_spans, spans.data(), ncols * sizeof(ColSpan));
    H2B_CUDA(cudaMemcpyAsync(d_spans, h_spans, ncols * sizeof(ColSpan), cudaMemcpyHostToDevice, ctx->stream));
    H2B_LAUNCH(ctx, k_assign_columns, ceil_div(total, 256), 256, 0, (const uint4*)d_vcol, d_spans, k, (u32)ncols, (uint4*)d_cols);
}

// MockProver's selector columns: q_c[r] = selector[s_c + r] for r < sel_len_c, zero elsewhere.  A column the walk left at a break
// has sel_len = len - 1: the break cell's selector is enabled at row 0 of the next column only (single_phase.rs:229-257 enable
// after the break), while the cell itself sits in both.
struct SelSpan {
    uint64_t start;
    uint64_t sel_len;
};
__global__ void __launch_bounds__(256) k_mock_selectors(const uint8_t* __restrict__ sel, const SelSpan* __restrict__ spans, u32 rows_log,
                                                        u32 ncols, uint64_t* __restrict__ q) {
    const size_t cell = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= ((size_t)ncols << rows_log)) return;
    const u32 c = (u32)(cell >> rows_log);
    const size_t r = cell & (((size_t)1 << rows_log) - 1);
    const SelSpan sp = spans[c];
    const bool on = r < sp.sel_len && __ldg(sel + sp.start + r) != 0;
    (on ? Fr::one() : Fr::zero()).store(q + 4 * cell);
}

// q_lookup[index[i]] = 1 (one gate column: the raw row of a virtual cell is its index).  bit 0 of *status: an index >= N;
// bit 1: an index >= max_rows (the row is not usable)
__global__ void __launch_bounds__(256) k_mock_lookup_selector(const uint64_t* __restrict__ index, size_t m, uint64_t N, uint64_t max_rows,
                                                              uint64_t* __restrict__ q, u32* __restrict__ status) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t idx = __ldg(index + i);
    const u32 bad = (idx < N ? 0u : 1u) | (idx < max_rows ? 0u : 2u);
    if (bad) {
        atomicOr(status, bad);
        return;
    }
    Fr::one().store(q + 4 * idx);
}

void mock_selectors_run(h2b_ctx* ctx, const void* d_selectors, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t ncols,
                        void* d_q) {
    H2B_REQUIRE(k <= 28, "mock_selectors: k out of range");
    H2B_REQUIRE(ncols >= 1, "mock_selectors: no gate columns");
    const size_t rows = (size_t)1 << k;
    const std::vector<ColSpan> spans = column_spans(N, break_points, nbp, rows, ncols);
    std::vector<SelSpan> sel(ncols);
    for (size_t c = 0; c < ncols; c++) {
        const bool broke = c + 1 < ncols && spans[c + 1].len > 0;
        sel[c] = SelSpan{spans[c].start, broke ? spans[c].len - 1 : spans[c].len};
    }
    SelSpan* d_spans = (SelSpan*)ctx->get(WS_MISC, ncols * sizeof(SelSpan));
    H2B_CUDA(cudaMemcpyAsync(d_spans, sel.data(), ncols * sizeof(SelSpan), cudaMemcpyHostToDevice, ctx->stream));  // pageable: staged now
    H2B_LAUNCH(ctx, k_mock_selectors, ceil_div(ncols * rows, 256), 256, 0, (const uint8_t*)d_selectors, (const SelSpan*)d_spans, k, (u32)ncols,
               (uint64_t*)d_q);
}

void mock_lookup_selector_run(h2b_ctx* ctx, const uint64_t* d_index, size_t m, size_t N, size_t max_rows, uint32_t k, void* d_q,
                              uint32_t* d_status) {
    H2B_REQUIRE(k <= 28, "mock_lookup_selector: k out of range");
    H2B_REQUIRE(max_rows <= ((size_t)1 << k), "mock_lookup_selector: max_rows > 2^k");
    H2B_CUDA(cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    H2B_CUDA(cudaMemsetAsync(d_q, 0, ((size_t)1 << k) * 32, ctx->stream));
    if (m == 0) return;
    H2B_LAUNCH(ctx, k_mock_lookup_selector, ceil_div(m, 256), 256, 0, d_index, m, (uint64_t)N, (uint64_t)max_rows, (uint64_t*)d_q, d_status);
}

// d_recs: N staging records of 72 bytes.  d_values (N x 32 B) receives what the prover's `batch_invert_assigned` yields:
// Zero -> 0, Trivial(x) -> x, Rational(n, d) -> n / d (d = 0 -> 0).  `stats` (device, 2 x u32, zeroed here): see above.
// invert: 0 = never (the caller knows there is no Rational cell), 1 = always (asynchronous).
void assigned_flatten_run(h2b_ctx* ctx, const void* d_recs, size_t N, void* d_values, u32* d_stats, int invert) {
    if (N == 0) return;
    uint64_t* den = (uint64_t*)ctx->get(WS_PROD, N * 32);
    H2B_CUDA(cudaMemsetAsync(d_stats, 0, 8, ctx->stream));
    H2B_LAUNCH(ctx, k_assigned_split, ceil_div(N, 256), 256, 0, (const uint64_t*)d_recs, N, (uint64_t*)d_values, den, d_stats);
    if (invert) {
        batch_invert_run(ctx, den, N);
        fr_mul_elementwise_run(ctx, d_values, den, N, d_values);
    }
}

void assign_lookups_run(h2b_ctx* ctx, const void* d_vals, size_t N, uint32_t k, size_t L, void* d_cols) {
    H2B_REQUIRE(k <= 28, "assign: k out of range");
    const size_t rows = (size_t)1 << k;
    if (L == 0) {
        if (N != 0) throw StatusError{H2B_ERR_LAYOUT, "assign_lookups: values present but no lookup advice columns (builder.rs:366)"};
        return;
    }
    if ((N + L - 1) / L > rows) throw StatusError{H2B_ERR_LAYOUT, "assign_lookups: range lookups would be assigned to unusable rows (builder.rs:368-372)"};
    size_t total = L * rows * 2;
    H2B_LAUNCH(ctx, k_assign_lookups, ceil_div(total, 256), 256, 0, (const uint4*)d_vals, N, k, (u32)L, (uint4*)d_cols);
}

void assign_lookups_indexed_run(h2b_ctx* ctx, const void* d_vals, size_t N, const uint64_t* d_index, size_t n_lookup, uint32_t k, size_t L,
                                void* d_cols, uint32_t* d_status) {
    H2B_REQUIRE(k <= 28, "assign: k out of range");
    const size_t rows = (size_t)1 << k;
    if (L == 0 && n_lookup != 0)
        throw StatusError{H2B_ERR_LAYOUT, "assign_lookups: values present but no lookup advice columns (builder.rs:366)"};
    if (L && (n_lookup + L - 1) / L > rows)
        throw StatusError{H2B_ERR_LAYOUT, "assign_lookups: range lookups would be assigned to unusable rows (builder.rs:368-372)"};
    H2B_CUDA(cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    if (L == 0) return;
    size_t total = L * rows * 2;
    H2B_LAUNCH(ctx, k_assign_lookups_indexed, ceil_div(total, 256), 256, 0, (const uint4*)d_vals, N, d_index, n_lookup, k, (u32)L,
               (uint4*)d_cols, d_status);
}

// d_den is inverted in place (batch_invert_run: zeros stay zero), then multiplied into the cells it belongs to
void apply_rational_run(h2b_ctx* ctx, void* d_values, size_t N, const uint64_t* d_index, void* d_den, size_t R, uint32_t* d_status) {
    H2B_CUDA(cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    if (R == 0) return;
    batch_invert_run(ctx, d_den, R);
    H2B_LAUNCH(ctx, k_apply_rational, ceil_div(R, 256), 256, 0, (uint64_t*)d_values, N, d_index, (const uint64_t*)d_den, R, d_status);
}

}  // namespace h2b
