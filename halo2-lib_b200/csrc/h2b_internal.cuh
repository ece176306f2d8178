// h2b_internal.cuh — context, workspace and launch helpers shared by the translation units of libh2b200.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include <array>
#include <algorithm>
#include <new>
#include <stdexcept>

#include "../../include/h2b200.h"

namespace h2b {

struct StatusError {
    int code;
    std::string msg;
};

#define H2B_CUDA(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess)                                                                      \
            throw h2b::StatusError{_e == cudaErrorMemoryAllocation ? H2B_ERR_OOM : H2B_ERR_CUDA,    \
                                   std::string(#expr) + ": " + cudaGetErrorString(_e)};             \
    } while (0)
#define H2B_REQUIRE(cond, msg)                                                   \
    do {                                                                         \
        if (!(cond)) throw h2b::StatusError{H2B_ERR_ARG, std::string(msg)};      \
    } while (0)

// grow-only device workspace slots (freed with the context)
enum WsSlot {
    WS_SCALARS = 0,   // staged scalars of host-pointer MSM calls (two of them for double buffering)
    WS_SCALARS2,
    WS_KEYS_A,
    WS_KEYS_B,
    WS_VALS_A,
    WS_VALS_B,
    WS_SORT_TMP,
    WS_OFFSETS,
    WS_BUCKETS,
    WS_PARTIALS,
    WS_BIGLIST,
    WS_REDUCE_A,
    WS_REDUCE_B,
    WS_POOL,
    WS_POOL2,
    WS_OUT,
    WS_BASES,         // ad-hoc bases staging
    WS_NTT_A,
    WS_NTT_B,
    WS_NTT_C,
    WS_NTT_D,
    WS_NTT_E,         // small (2^k) buffers of the fused lagrange -> coeff -> extended batch
    WS_NTT_F,
    WS_NTT_G,
    WS_ASSIGN_IN,
    WS_ASSIGN_OUT,
    WS_MISC,
    WS_MISC2,
    WS_PROD,          // product-column scratch (numerators, denominators, power tables)
    WS_CHECK_FLAGS,   // constraint check: one flag byte per checked cell, then the tile counts of the reports
    WS_CHECK_TABLES,  // constraint check: omega powers and the hash table of the sigma decode
    WS_COUNT
};

struct NttPlan;

}  // namespace h2b

struct h2b_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    cudaStream_t copy_stream2 = nullptr;  // device-to-host leg of the pipelined batch NTT entry points
    cudaStream_t side_stream = nullptr;   // h2b_ctx_side_begin / _end / _join: work that runs beside the main stream
    cudaStream_t side_saved = nullptr;    // the main stream while the side stream is current
    int side_saved_lane = 0;              // the side queue works in the workspace set of lane 1 (its own scratch buffers)
    cudaEvent_t side_ev[2] = {nullptr, nullptr};
    cudaEvent_t pipe_ev[3][3] = {};       // [buffer][uploaded, computed, downloaded]
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    int sm_count = 132;
    mutable std::mutex mu;
    std::string err;
    uint64_t launches = 0;
    bool ntt_attr_set = false;
    bool sort_attr_set = false;  // MSM sort kernels allowed their larger dynamic shared memory (msm_run_group)
    int opt_ntt_ctas = 0;        // h2b_ctx_set_option("ntt.max_ctas_per_sm"): 0 = as many as fit, 1 or 2 = background transform (see ntt_run)
    int opt_msm_group = 0;       // "msm.batch_group": MSMs of a batch call that share one sort / accumulate / reduce pipeline (0 = by size)
    int opt_lookup_backward = 0; // "lookup.leftover_order": 0 = front to back (PSE / axiom walk), 1 = zcash (pop from the back)
    void* peer = nullptr;  // PeerState (peer.cu): NVLink mailboxes of the multi-GPU all-reduce
    std::vector<h2b_ctx*> members;  // device group (h2b_ctx_create_multi): members[0] == this, the others are private
    bool reduce_counter_zeroed = false;
    void* reduce_counter_ptr = nullptr;
    struct Buf {
        void* p = nullptr;
        size_t cap = 0;
    };
    // MSM lanes: independent (stream, workspace) sets so that the latency-bound tail of one MSM (bucket
    // reduction: a few CTAs) overlaps the throughput-bound phases of the next MSM of the same batch
    static constexpr int NLANES = 3;
    cudaStream_t lane_stream[NLANES] = {nullptr, nullptr, nullptr};
    cudaStream_t lane_tail[NLANES] = {nullptr, nullptr, nullptr};     // high priority: the bucket reduction of the lane's MSM
    cudaEvent_t lane_acc[NLANES] = {nullptr, nullptr, nullptr};       // accumulation of the lane's MSM enqueued
    cudaEvent_t lane_tail_done[NLANES] = {nullptr, nullptr, nullptr};
    bool in_lane = false;                                             // the current stream is lane_stream[cur_lane]
    cudaEvent_t lane_done[NLANES] = {nullptr, nullptr, nullptr};
    cudaEvent_t lane_ready[NLANES] = {nullptr, nullptr, nullptr};     // staging buffer filled (host batch API)
    cudaEvent_t lane_consumed[NLANES] = {nullptr, nullptr, nullptr};  // staging buffer read by the MSM sort
    cudaEvent_t fork_ev = nullptr;
    int cur_lane = 0;  // workspace set used by get()
    Buf ws[NLANES][h2b::WS_COUNT];
    Buf pinned[3];
    std::map<std::array<uint64_t, 5>, h2b::NttPlan*> ntt_plans;

    // optional per-kernel device timing (h2b_profile_*): event pairs around launches whose name matches
    std::string prof_filter;  // empty = off, "*" = every kernel, else substring of the kernel name
    struct ProfRec {
        const char* name;
        cudaEvent_t a, b;
        cudaStream_t stream;
    };
    std::vector<ProfRec> prof_recs;
    std::vector<cudaEvent_t> prof_pool;
    bool prof_match(const char* name) const {
        return !prof_filter.empty() && (prof_filter == "*" || std::string(name).find(prof_filter) != std::string::npos);
    }
    cudaEvent_t prof_event();

    // grow-only; growing synchronises the device first (a kernel may still read the old block)
    void* get(int slot, size_t bytes);
    void* get_pinned(int slot, size_t bytes);
};

struct h2b_srs {
    uint32_t k = 0;
    size_t begin = 0, count = 0;
    int c = 0, W = 0;
    void* table[2] = {nullptr, nullptr};  // [basis] -> W x count affine points: table[w*count + i] = 2^(c*w) * P_i
    std::vector<h2b_srs*> parts;          // device group: one shard handle per member device (tables above unused)
};

namespace h2b {

#define H2B_LAUNCH(ctx, kernel, grid, block, smem, ...)                          \
    do {                                                                         \
        const bool _prof = (ctx)->prof_match(#kernel);                           \
        cudaEvent_t _ea = nullptr, _eb = nullptr;                                \
        if (_prof) {                                                             \
            _ea = (ctx)->prof_event();                                           \
            _eb = (ctx)->prof_event();                                           \
            H2B_CUDA(cudaEventRecord(_ea, (ctx)->stream));                       \
        }                                                                        \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);         \
        (ctx)->launches++;                                                       \
        H2B_CUDA(cudaGetLastError());                                            \
        if (_prof) {                                                             \
            H2B_CUDA(cudaEventRecord(_eb, (ctx)->stream));                       \
            (ctx)->prof_recs.push_back({#kernel, _ea, _eb, (ctx)->stream});                     \
        }                                                                        \
    } while (0)

// Runs the body of a C entry point under the context lock with the context's device current; maps every failure to a
// status code and h2b_last_error()'s message.  No exception leaves an entry point.
template <class Fn>
static int guarded(h2b_ctx* ctx, Fn&& body) {
    if (!ctx) return H2B_ERR_ARG;
    std::lock_guard<std::mutex> lock(ctx->mu);
    try {
        H2B_CUDA(cudaSetDevice(ctx->device));
        body();
        return H2B_OK;
    } catch (const StatusError& e) {
        ctx->err = e.msg;
        return e.code;
    } catch (const std::bad_alloc&) {
        ctx->err = "host allocation failed";
        return H2B_ERR_OOM;
    } catch (const std::exception& e) {
        ctx->err = e.what();
        return H2B_ERR_CUDA;
    } catch (...) {
        ctx->err = "unknown failure";
        return H2B_ERR_CUDA;
    }
}

static inline unsigned ceil_div(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }
static inline int ceil_log2(size_t n) {
    int l = 0;
    while (((size_t)1 << l) < n) l++;
    return l;
}

// ---- msm.cu
int msm_choose_c_fixed(size_t n);
void msm_build_table(h2b_ctx* ctx, const void* d_bases, size_t count, int c, int W, void* d_table);
// table mode: q = W (one bucket set), table = W x n affine; ad-hoc mode: q = 1, table = n affine
void msm_run(h2b_ctx* ctx, const void* d_table, size_t n, int c, int W, int q, const void* d_scalars, void* d_out,
             cudaEvent_t after_digits = nullptr);
// m MSMs of one size through ONE sort / accumulate / bucket-reduction pipeline (m <= 16; tabulated bases unless m == 1)
void msm_run_group(h2b_ctx* ctx, const void* const* d_tables, size_t n, int c, int W, int q, const void* const* d_scalars, size_t m,
                   void* d_out, cudaEvent_t after_digits = nullptr);
size_t msm_group_size(const h2b_ctx* ctx, size_t n, size_t m, int W);  // MSMs per pipeline for a batch of m
// m MSMs over tabulated bases: cut into groups (msm_run_group) that are dealt to the context's lanes; joins on ctx->stream
void msm_run_batch(h2b_ctx* ctx, const void* const* d_tables, size_t n, int c, int W, const void* const* d_scalars, size_t m, void* d_out);
void g1_sum_run(h2b_ctx* ctx, const void* d_points, size_t m, void* d_out);
void g1_normalize_run(h2b_ctx* ctx, void* d_points, size_t m);
void g1_fixed_base_mul_run(h2b_ctx* ctx, const uint64_t base_xy[8], const void* d_scalars, size_t n, void* d_out);
void field_op_run(h2b_ctx* ctx, int field, int op, const void* a, const void* b, size_t n, void* out);
// ---- ntt.cu
// in-place forward transform with arbitrary root; flags: see ntt.cu
void ntt_run(h2b_ctx* ctx, const void* d_src, size_t n_src, void* d_dst, uint32_t log_n, const uint64_t omega[4],
             int inverse_scale, int coset_mode);
void ntt_free_plans(h2b_ctx* ctx);
void domain_omega(uint32_t k, uint64_t out[4], bool inverse);
// ---- assign.cu
void assign_columns_run(h2b_ctx* ctx, const void* d_vcol, size_t N, const uint64_t* break_points, size_t nbp,
                        uint32_t k, size_t ncols, void* d_cols);
void assigned_flatten_run(h2b_ctx* ctx, const void* d_recs, size_t N, void* d_values, uint32_t* d_stats, int invert);
void assign_lookups_run(h2b_ctx* ctx, const void* d_vals, size_t N, uint32_t k, size_t L, void* d_cols);
// halo2-base form of the witness (asynchronous; violations land in *d_status, which both zero first)
void apply_rational_run(h2b_ctx* ctx, void* d_values, size_t N, const uint64_t* d_index, void* d_den, size_t R, uint32_t* d_status);
// MockProver on halo2-base's keygen data (include/h2b200.h, "MockProver for a halo2-base builder")
void mock_selectors_run(h2b_ctx* ctx, const void* d_selectors, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t ncols,
                        void* d_q);
void mock_lookup_selector_run(h2b_ctx* ctx, const uint64_t* d_index, size_t m, size_t N, size_t max_rows, uint32_t k, void* d_q,
                              uint32_t* d_status);
void assign_lookups_indexed_run(h2b_ctx* ctx, const void* d_vals, size_t N, const uint64_t* d_index, size_t n_lookup, uint32_t k, size_t L,
                                void* d_cols, uint32_t* d_status);
// ---- peer.cu
void peer_create(h2b_ctx* ctx, int rank, int nranks, uint8_t* handle_out);
void peer_connect(h2b_ctx* ctx, const uint8_t* handles);
void peer_allreduce(h2b_ctx* ctx, void* d_points, size_t m);
void peer_destroy(h2b_ctx* ctx);
bool peer_connected(const h2b_ctx* ctx);
void peer_connect_local(const std::vector<h2b_ctx*>& members);  // in-process group: direct peer mappings
// ---- quotient.cu
void flex_gate_fold_run(h2b_ctx* ctx, const void* d_q_ext, const void* d_a_ext, const uint64_t y[4], uint32_t k, uint32_t ext_k,
                        void* d_acc);
void divide_by_vanishing_run(h2b_ctx* ctx, void* d_values, uint32_t k, uint32_t ext_k);
void quotient_graph_run(h2b_ctx* ctx, const h2b_graph* g, uint32_t k, uint32_t ext_k, void* d_values);
void lookup_fold_run(h2b_ctx* ctx, const h2b_graph* g, const void* d_z, const void* d_pin, const void* d_ptab, const void* d_l0,
                     const void* d_l_last, const void* d_l_active, uint32_t k, uint32_t ext_k, void* d_values);
void permutation_fold_run(h2b_ctx* ctx, const void* const* d_z, size_t n_sets, const void* const* d_columns, const void* const* d_sigma,
                          size_t n_cols, size_t chunk_len, const void* d_l0, const void* d_l_last, const void* d_l_active,
                          const uint64_t beta[4], const uint64_t gamma[4], const uint64_t y[4], uint32_t blinding_factors, uint32_t k,
                          uint32_t ext_k, void* d_values);
// ---- lookup.cu (returns true when an input value is missing from the table)
uint32_t* permute_expression_pair_enqueue(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                          void* d_permuted_input, void* d_permuted_table);  // enqueue only; returns the device verdict word
bool permute_expression_pair_run(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                 void* d_permuted_input, void* d_permuted_table);
// the canonical sort of one column of n elements: out = src sorted by canonical value, out_canon = those canonical values;
// scratch holds sort_column_scratch(n, sort_ctas) bytes, sort_ctas = sort_column_ctas(ctx, n) (the cooperative grid)
int sort_column_ctas(h2b_ctx* ctx, uint32_t n);
size_t sort_column_scratch(uint32_t n, int sort_ctas);
void sort_column(h2b_ctx* ctx, const uint64_t* d_src, uint32_t n, uint64_t* d_out, uint64_t* d_out_canon, char* scratch, int sort_ctas);
// the same stable sort on n 256-bit integer keys (4 little-endian uint64 each, not field elements): d_perm[i] = the id of the
// i-th smallest key, ties in the order of d_init (the identity when null); scratch holds sort_keys_scratch(n, sort_ctas) bytes
size_t sort_keys_scratch(uint32_t n, int sort_ctas);
void sort_keys(h2b_ctx* ctx, const uint64_t* d_keys, uint32_t n, const uint32_t* d_init, uint32_t* d_perm, char* scratch, int sort_ctas);
// d_out[i] = d_in[0] + .. + d_in[i - 1] (uint32); scratch holds exclusive_scan_scratch(n) bytes
size_t exclusive_scan_scratch(uint32_t n);
void exclusive_scan(h2b_ctx* ctx, const uint32_t* d_in, uint32_t n, uint32_t* d_out, char* scratch);
// ---- ntt.cu: omega^r = lo[r mod 2^h] * hi[r >> h] for the 2^k domain root (the power tables of its NTT plan)
void domain_power_tables(h2b_ctx* ctx, uint32_t k, const void** lo, const void** hi, int* h);
// ---- keygen.cu (include/h2b200.h, "keygen of a halo2-base builder")
void keygen_copies_run(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                       const uint64_t* d_lookup_index, size_t n_lookup, const uint64_t* d_pairs, size_t M, const void* d_consts,
                       const uint64_t* d_const_index, size_t Mc, void* d_c, void* d_edges, uint32_t* status);
void keygen_instance_edges_run(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                               size_t usable, size_t I, const size_t* n_index, const uint64_t* d_index, void* d_edges, uint32_t* status);
void keygen_sigma_map_run(h2b_ctx* ctx, const void* d_edges, size_t E, size_t n_cols, uint32_t k, void* d_map);
void keygen_sigma_values_run(h2b_ctx* ctx, const void* d_map, size_t n_cols, uint32_t k, void* d_sigma);
// ---- check.cu (MockProver::verify's checks; reports of max_report + 1 words per item, see include/h2b200.h)
void check_graph_run(h2b_ctx* ctx, const h2b_graph* g, uint32_t k, size_t rows, size_t max_report, void* d_report);
void check_lookup_run(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, size_t rows, size_t max_report, void* d_report);
void permutation_decode_run(h2b_ctx* ctx, const void* const* d_sigma, size_t n_cols, uint32_t k, void* d_map, size_t max_report,
                            void* d_reports);
void check_copies_run(h2b_ctx* ctx, const void* const* d_columns, const void* d_map, size_t n_cols, uint32_t k, size_t max_report,
                      void* d_reports);
void check_equalities_run(h2b_ctx* ctx, const void* d_cells, size_t N, const uint64_t* d_pairs, size_t m, size_t max_report, void* d_report,
                          uint32_t* d_status);
void check_constants_run(h2b_ctx* ctx, const void* d_cells, size_t N, const void* d_consts, const uint64_t* d_index, size_t m,
                         size_t max_report, void* d_report, uint32_t* d_status);
void count_distinct_run(h2b_ctx* ctx, const void* d_values, size_t m, uint32_t* d_count);
// ---- selectors.cu (host output, synchronises)
void selector_conflicts_run(h2b_ctx* ctx, const void* const* d_cols, size_t S, uint32_t k, uint8_t* conflicts);
// ---- srs.cu
void g_to_lagrange_run(h2b_ctx* ctx, const void* d_g, uint32_t k, void* d_g_lagrange);
void srs_setup_run(h2b_ctx* ctx, const uint64_t tau[4], const uint64_t base_xy[8], uint32_t k, void* d_g, void* d_g_lagrange);
size_t g1_count_off_curve_run(h2b_ctx* ctx, const void* d_points, size_t n);
size_t g1_decompress_run(h2b_ctx* ctx, const void* d_bytes, size_t n, void* d_out_xy);
void g1_compress_run(h2b_ctx* ctx, const void* d_xy, size_t n, void* d_bytes);
// ---- poly.cu
void eval_polynomial_run(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t x[4], void* d_out);
void eval_polynomial_batch_run(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* xs, size_t m, size_t n, void* d_out);
void kate_division_run(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t z[4], void* d_q);
void kate_division_multi_run(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t* points, size_t m, const uint64_t* weights, void* d_q);
void poly_lincomb_run(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* scalars, size_t m, size_t n, void* d_out);
// ---- scan.cu
void batch_invert_run(h2b_ctx* ctx, void* d_a, size_t n);
// d_start != nullptr: the seed is read from device memory (the previous permutation set's closing value) instead of `start`
void grand_product_run(h2b_ctx* ctx, const void* d_f, const uint64_t start[4], size_t n, void* d_z, const void* d_start = nullptr);
void eval_rational_batched_run(h2b_ctx* ctx, const void* d_num, const void* d_den, size_t n, void* d_out);
// ---- prover.cu
void permutation_product_run(h2b_ctx* ctx, const void* const* d_columns, const void* const* d_sigma, size_t n_cols, size_t first_col,
                             const uint64_t beta[4], const uint64_t gamma[4], uint32_t k, uint32_t blinding_factors,
                             const void* d_start, void* d_z);
void lookup_product_run(h2b_ctx* ctx, const void* d_in, const void* d_tab, const void* d_pin, const void* d_ptab, const uint64_t beta[4],
                        const uint64_t gamma[4], uint32_t k, uint32_t blinding_factors, void* d_z);
void fr_mul_elementwise_run(h2b_ctx* ctx, const void* d_a, const void* d_b, size_t n, void* d_out);

}  // namespace h2b
