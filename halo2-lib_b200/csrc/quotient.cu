// quotient.cu — first slice of the quotient evaluation h(X) on the extended domain (SURVEY.md §8(f) rank 1):
// the custom-gate term of halo2-base's single vertical gate
//     q * (a + b * c - out)      with a, b, c, out = the SAME advice column at rotations 0, 1, 2, 3
// (halo2-base/src/gates/flex_gate/mod.rs:80-91), folded into the running combination the prover keeps per
// extended-domain row:  acc[i] <- acc[i] * y + q[i] * (a[i] + a[i + s] * a[i + 2s] - a[i + 3s]),
// s = 2^(extended_k - k) (a rotation by one row of the 2^k domain is a shift by s rows of the extended coset
// domain; indices wrap).  Pointwise: 3 products per row; HBM traffic 32 B x (q, acc in, acc out, a + 3 rotated reads
// that hit L2).
#include "h2b_internal.cuh"
#include "field.cuh"

namespace h2b {

__global__ void __launch_bounds__(256) k_flex_gate_fold(const uint64_t* __restrict__ q, const uint64_t* __restrict__ a, Fr y,
                                                        u32 ext_k, u32 shift, uint64_t* __restrict__ acc) {
    const size_t n = (size_t)1 << ext_k, mask = n - 1;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t s = (size_t)1 << shift;
    Fr a0 = Fr::load_nc(a + 4 * i), a1 = Fr::load_nc(a + 4 * ((i + s) & mask)), a2 = Fr::load_nc(a + 4 * ((i + 2 * s) & mask)),
       a3 = Fr::load_nc(a + 4 * ((i + 3 * s) & mask));
    Fr gate = Fr::load_nc(q + 4 * i) * (a0 + a1 * a2 - a3);
    (Fr::load(acc + 4 * i) * y + gate).store(acc + 4 * i);
}

void flex_gate_fold_run(h2b_ctx* ctx, const void* d_q_ext, const void* d_a_ext, const uint64_t y[4], uint32_t k, uint32_t ext_k,
                        void* d_acc) {
    H2B_REQUIRE(ext_k >= k && ext_k <= 28, "flex_gate: extended_k out of range");
    Fr yy;
    memcpy(&yy, y, sizeof(Fr));
    H2B_LAUNCH(ctx, k_flex_gate_fold, ceil_div((size_t)1 << ext_k, 256), 256, 0, (const uint64_t*)d_q_ext, (const uint64_t*)d_a_ext, yy,
               ext_k, ext_k - k, (uint64_t*)d_acc);
}

}  // namespace h2b

// =====================================================================================================================
// General quotient evaluation: the GraphEvaluator interpreter (graph.cuh) and the permutation / lookup argument terms of
// halo2-axiom 0.5.3 `plonk/evaluation.rs::Evaluator::evaluate_h` (not vendored; restated from the upstream algorithm).
// One thread per extended-domain row; every term is pointwise, so the kernels are HBM-bound:
// 32 B per column read per row (rotated reads of the same column hit L2) + 64 B for `values` in / out.
#include "fr_domain_consts.inc"
#include "graph.cuh"

namespace h2b {

__global__ void __launch_bounds__(128) k_quotient_graph(GraphDev g, u32 ext_k, u32 rshift, uint64_t* __restrict__ values) {
    const size_t n = (size_t)1 << ext_k, idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    Fr inter[H2B_GRAPH_MAX_CALCULATIONS];
    const Fr prev = Fr::load(values + 4 * idx);
    graph_eval(g, idx, n - 1, rshift, prev, inter).store(values + 4 * idx);
}

__global__ void __launch_bounds__(128) k_lookup_fold(GraphDev g, const uint64_t* __restrict__ z, const uint64_t* __restrict__ pin,
                                                     const uint64_t* __restrict__ ptab, const uint64_t* __restrict__ l0,
                                                     const uint64_t* __restrict__ l_last, const uint64_t* __restrict__ l_active,
                                                     u32 ext_k, u32 rshift, uint64_t* __restrict__ values) {
    const size_t n = (size_t)1 << ext_k, mask = n - 1, idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    Fr inter[H2B_GRAPH_MAX_CALCULATIONS];
    const Fr table_value = graph_eval(g, idx, mask, rshift, Fr::zero(), inter);
    const Fr zc = Fr::load_nc(z + 4 * idx), zn = Fr::load_nc(z + 4 * rot_idx(idx, 1, rshift, mask));
    const Fr a = Fr::load_nc(pin + 4 * idx), ap = Fr::load_nc(pin + 4 * rot_idx(idx, -1, rshift, mask));
    const Fr s = Fr::load_nc(ptab + 4 * idx);
    const Fr v0 = Fr::load_nc(l0 + 4 * idx), vl = Fr::load_nc(l_last + 4 * idx), va = Fr::load_nc(l_active + 4 * idx);
    const Fr a_minus_s = a - s;
    Fr v = Fr::load(values + 4 * idx);
    v = v * g.y + (Fr::one() - zc) * v0;
    v = v * g.y + (zc.sqr() - zc) * vl;
    v = v * g.y + (zn * (a + g.beta) * (s + g.gamma) - zc * table_value) * va;
    v = v * g.y + a_minus_s * v0;
    v = v * g.y + a_minus_s * (a - ap) * va;
    v.store(values + 4 * idx);
}

struct PermDev {
    const uint64_t* const* z;        // n_sets
    const uint64_t* const* columns;  // n_cols
    const uint64_t* const* sigma;    // n_cols
    const uint64_t* omega_pow2;      // [j] = extended_omega^(2^j), j < ext_k
    const uint64_t* pow_lo;          // [i] = extended_omega^i, i < 2^lo_bits
    const uint64_t* pow_hi;          // [j] = beta * zeta * extended_omega^(j << lo_bits)
    u32 n_sets, n_cols, chunk_len, lo_bits;
    int last_rotation;
    Fr beta, gamma, y, zeta, delta;
};

// the two tables that turn beta * zeta * extended_omega^idx (= beta * X at row idx) into one product per row
__global__ void __launch_bounds__(256) k_omega_tables(PermDev p, u32 ext_k, uint64_t* __restrict__ lo, uint64_t* __restrict__ hi) {
    const u32 idx = blockIdx.x * blockDim.x + threadIdx.x, n_lo = 1u << p.lo_bits, hi_bits = ext_k - p.lo_bits;
    if (idx < n_lo) {
        Fr r = Fr::one();
        for (u32 j = 0; j < p.lo_bits; j++)
            if ((idx >> j) & 1) r = r * Fr::load_nc(p.omega_pow2 + 4 * (size_t)j);
        r.store(lo + 4 * (size_t)idx);
    } else if (idx - n_lo < (1u << hi_bits)) {
        const u32 h = idx - n_lo;
        Fr r = p.beta * p.zeta;
        for (u32 j = 0; j < hi_bits; j++)
            if ((h >> j) & 1) r = r * Fr::load_nc(p.omega_pow2 + 4 * (size_t)(p.lo_bits + j));
        r.store(hi + 4 * (size_t)h);
    }
}

__global__ void __launch_bounds__(128) k_permutation_fold(PermDev p, const uint64_t* __restrict__ l0, const uint64_t* __restrict__ l_last,
                                                          const uint64_t* __restrict__ l_active, u32 ext_k, u32 rshift,
                                                          uint64_t* __restrict__ values) {
    const size_t n = (size_t)1 << ext_k, mask = n - 1, idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const size_t r_next = rot_idx(idx, 1, rshift, mask), r_last = rot_idx(idx, p.last_rotation, rshift, mask);
    const Fr v0 = Fr::load_nc(l0 + 4 * idx), vl = Fr::load_nc(l_last + 4 * idx), va = Fr::load_nc(l_active + 4 * idx);
    Fr v = Fr::load(values + 4 * idx);
    {
        const Fr z0 = Fr::load_nc(p.z[0] + 4 * idx);
        v = v * p.y + (Fr::one() - z0) * v0;
        const Fr zl = Fr::load_nc(p.z[p.n_sets - 1] + 4 * idx);
        v = v * p.y + (zl.sqr() - zl) * vl;
    }
#pragma unroll 1
    for (u32 s = 1; s < p.n_sets; s++)
        v = v * p.y + (Fr::load_nc(p.z[s] + 4 * idx) - Fr::load_nc(p.z[s - 1] + 4 * r_last)) * v0;
    // current_delta = beta * zeta * extended_omega^idx  (= beta * X at this row), then *= DELTA per column
    Fr cur = Fr::load_nc(p.pow_hi + 4 * (idx >> p.lo_bits)) * Fr::load_nc(p.pow_lo + 4 * (idx & (((size_t)1 << p.lo_bits) - 1)));
    u32 col = 0;
#pragma unroll 1
    for (u32 s = 0; s < p.n_sets; s++) {
        Fr left = Fr::load_nc(p.z[s] + 4 * r_next), right = Fr::load_nc(p.z[s] + 4 * idx);
#pragma unroll 1
        for (u32 j = 0; j < p.chunk_len && col < p.n_cols; j++, col++) {
            const Fr val = Fr::load_nc(p.columns[col] + 4 * idx);
            left = left * (val + p.beta * Fr::load_nc(p.sigma[col] + 4 * idx) + p.gamma);
            right = right * (val + cur + p.gamma);
            cur = cur * p.delta;
        }
        v = v * p.y + (left - right) * va;
    }
    v.store(values + 4 * idx);
}

// EvaluationDomain::divide_by_vanishing_poly: t(X) = X^n - 1 takes only 2^(ext_k - k) distinct values on the coset
// zeta * <extended_omega> (period 2^(ext_k - k) in the row index): t_inv[j] = 1 / (zeta^n * (extended_omega^n)^j - 1).
__global__ void k_vanishing_table(Fr zeta, Fr ext_omega, u32 k, u32 period, uint64_t* __restrict__ t_inv) {
    const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= period) return;
    Fr zn = zeta, step = ext_omega;
    for (u32 i = 0; i < k; i++) { zn = zn.sqr(); step = step.sqr(); }  // ^n, n = 2^k
    Fr cur = zn;
    for (u32 b = 0; (j >> b) != 0; b++) {
        if ((j >> b) & 1) cur = cur * step;
        step = step.sqr();
    }
    (cur - Fr::one()).inv_bgcd().store(t_inv + 4 * (size_t)j);
}
__global__ void __launch_bounds__(256) k_divide_by_vanishing(const uint64_t* __restrict__ t_inv, u32 ext_k, u32 period_mask,
                                                             uint64_t* __restrict__ values) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >> ext_k) return;
    (Fr::load(values + 4 * i) * Fr::load_nc(t_inv + 4 * (i & period_mask))).store(values + 4 * i);
}

static Fr fr_from(const uint64_t x[4]) {
    Fr r;
    memcpy(&r, x, sizeof(Fr));
    return r;
}

// checks a program the way the device will walk it; throws H2B_ERR_ARG on anything out of range
static void graph_validate(const h2b_graph* g) {
    H2B_REQUIRE(g, "graph: null pointer");
    H2B_REQUIRE(g->n_calculations <= H2B_GRAPH_MAX_CALCULATIONS, "graph: too many calculations");
    H2B_REQUIRE(g->program || g->program_words == 0, "graph: null program");
    H2B_REQUIRE((g->constants || !g->n_constants) && (g->rotations || !g->n_rotations) && (g->fixed || !g->n_fixed) &&
                    (g->advice || !g->n_advice) && (g->instance || !g->n_instance) && (g->challenges || !g->n_challenges),
                "graph: null table");
    H2B_REQUIRE(g->n_constants < 65536 && g->n_fixed < 65536 && g->n_advice < 65536 && g->n_instance < 65536 &&
                    g->n_challenges < 65536 && g->n_rotations < 4096, "graph: table too large");
    auto check_src = [&](u32 src, u32 t) {
        const u32 kind = src & 15u, index = (src >> 4) & 0xffffu, slot = src >> 20;
        switch (kind) {
            case H2B_SRC_CONSTANT: H2B_REQUIRE(index < g->n_constants, "graph: constant index out of range"); break;
            case H2B_SRC_INTERMEDIATE: H2B_REQUIRE(index < t, "graph: intermediate used before it is computed"); break;
            case H2B_SRC_FIXED: H2B_REQUIRE(index < g->n_fixed && slot < g->n_rotations, "graph: fixed query out of range"); break;
            case H2B_SRC_ADVICE: H2B_REQUIRE(index < g->n_advice && slot < g->n_rotations, "graph: advice query out of range"); break;
            case H2B_SRC_INSTANCE: H2B_REQUIRE(index < g->n_instance && slot < g->n_rotations, "graph: instance query out of range"); break;
            case H2B_SRC_CHALLENGE: H2B_REQUIRE(index < g->n_challenges, "graph: challenge index out of range"); break;
            case H2B_SRC_BETA: case H2B_SRC_GAMMA: case H2B_SRC_THETA: case H2B_SRC_Y: case H2B_SRC_PREVIOUS: break;
            default: throw StatusError{H2B_ERR_ARG, "graph: unknown value source"};
        }
    };
    size_t pc = 0;
    auto next = [&]() {
        H2B_REQUIRE(pc < g->program_words, "graph: program truncated");
        return g->program[pc++];
    };
    for (u32 t = 0; t < g->n_calculations; t++) {
        const u32 op = next();
        H2B_REQUIRE(op <= H2B_CALC_STORE, "graph: unknown opcode");
        if (op == H2B_CALC_HORNER) {
            check_src(next(), t);
            check_src(next(), t);
            const u32 np = next();
            H2B_REQUIRE(np <= g->program_words, "graph: horner part count");
            for (u32 j = 0; j < np; j++) check_src(next(), t);
        } else {
            check_src(next(), t);
            if (op <= H2B_CALC_MUL) check_src(next(), t);
        }
    }
    H2B_REQUIRE(pc == g->program_words, "graph: trailing program words");
    check_src(g->result, g->n_calculations);
}

// packs program + tables into one device blob (slot WS_MISC) and returns the device view (declared in graph.cuh)
// `Store(x)` calculations (every column query of an expression becomes one) are resolved on the host: users of the
// intermediate read x directly and the Store becomes a no-op, which halves the local-memory traffic of the interpreter
// for halo2-base's gate (5 of its 10 calculations are Stores).
static std::vector<u32> graph_resolve_stores(const h2b_graph* g, u32* result) {
    std::vector<u32> out, alias(g->n_calculations, 0);
    std::vector<char> has(g->n_calculations, 0);
    auto res = [&](u32 src) {
        const u32 kind = src & 15u, index = (src >> 4) & 0xffffu;
        return (kind == H2B_SRC_INTERMEDIATE && has[index]) ? alias[index] : src;
    };
    size_t pc = 0;
    for (u32 t = 0; t < g->n_calculations; t++) {
        const u32 op = g->program[pc++];
        if (op == H2B_CALC_STORE) {
            alias[t] = res(g->program[pc++]);
            has[t] = 1;
            out.push_back(CALC_NOP);
        } else if (op == H2B_CALC_HORNER) {
            const u32 np = g->program[pc + 2];
            out.push_back(op);
            out.push_back(res(g->program[pc]));
            out.push_back(res(g->program[pc + 1]));
            out.push_back(np);
            for (u32 j = 0; j < np; j++) out.push_back(res(g->program[pc + 3 + j]));
            pc += 3 + np;
        } else {
            out.push_back(op);
            out.push_back(res(g->program[pc++]));
            if (op <= H2B_CALC_MUL) out.push_back(res(g->program[pc++]));
        }
    }
    *result = res(g->result);
    return out;
}

GraphDev graph_upload(h2b_ctx* ctx, const h2b_graph* g) {
    graph_validate(g);
    u32 result = 0;
    const std::vector<u32> program = graph_resolve_stores(g, &result);
    auto al = [](size_t x) { return (x + 31) & ~(size_t)31; };
    const size_t o_prog = 0, o_const = al(o_prog + 4 * (program.size() + 1)), o_rot = al(o_const + 32 * g->n_constants),
                 o_fix = al(o_rot + 4 * g->n_rotations), o_adv = al(o_fix + 8 * g->n_fixed), o_ins = al(o_adv + 8 * g->n_advice),
                 o_ch = al(o_ins + 8 * g->n_instance), total = al(o_ch + 32 * g->n_challenges) + 32;
    std::vector<char> host(total, 0);
    if (!program.empty()) memcpy(host.data() + o_prog, program.data(), 4 * program.size());
    if (g->n_constants) memcpy(host.data() + o_const, g->constants, 32 * g->n_constants);
    if (g->n_rotations) memcpy(host.data() + o_rot, g->rotations, 4 * g->n_rotations);
    if (g->n_fixed) memcpy(host.data() + o_fix, g->fixed, 8 * g->n_fixed);
    if (g->n_advice) memcpy(host.data() + o_adv, g->advice, 8 * g->n_advice);
    if (g->n_instance) memcpy(host.data() + o_ins, g->instance, 8 * g->n_instance);
    if (g->n_challenges) memcpy(host.data() + o_ch, g->challenges, 32 * g->n_challenges);
    for (size_t i = 0; i < g->n_fixed; i++) H2B_REQUIRE(g->fixed[i], "graph: null fixed column");
    for (size_t i = 0; i < g->n_advice; i++) H2B_REQUIRE(g->advice[i], "graph: null advice column");
    for (size_t i = 0; i < g->n_instance; i++) H2B_REQUIRE(g->instance[i], "graph: null instance column");
    char* d = (char*)ctx->get(WS_MISC, total);
    // pageable source: the runtime stages it before returning, so `host` may die at the end of this function
    H2B_CUDA(cudaMemcpyAsync(d, host.data(), total, cudaMemcpyHostToDevice, ctx->stream));
    GraphDev r;
    r.program = (const u32*)(d + o_prog);
    r.n_calc = g->n_calculations;
    r.result = result;
    r.constants = (const uint64_t*)(d + o_const);
    r.rotations = (const int32_t*)(d + o_rot);
    r.fixed = (const uint64_t* const*)(d + o_fix);
    r.advice = (const uint64_t* const*)(d + o_adv);
    r.instance = (const uint64_t* const*)(d + o_ins);
    r.challenges = (const uint64_t*)(d + o_ch);
    r.beta = fr_from(g->beta);
    r.gamma = fr_from(g->gamma);
    r.theta = fr_from(g->theta);
    r.y = fr_from(g->y);
    return r;
}

static void check_domain(uint32_t k, uint32_t ext_k) { H2B_REQUIRE(ext_k >= k && ext_k <= 28, "quotient: extended_k out of range"); }

void divide_by_vanishing_run(h2b_ctx* ctx, void* d_values, uint32_t k, uint32_t ext_k) {
    check_domain(k, ext_k);
    H2B_REQUIRE(ext_k > k, "divide_by_vanishing_poly: the extended domain must be larger than the domain (t vanishes on it otherwise)");
    const u32 period = 1u << (ext_k - k);
    uint64_t* t_inv = (uint64_t*)ctx->get(WS_MISC2, 32 * (size_t)period);
    H2B_LAUNCH(ctx, k_vanishing_table, ceil_div(period, 64), 64, 0, fr_from(FR_ZETA_U64), fr_from(FR_OMEGA[ext_k]), k, period, t_inv);
    H2B_LAUNCH(ctx, k_divide_by_vanishing, ceil_div((size_t)1 << ext_k, 256), 256, 0, t_inv, ext_k, period - 1, (uint64_t*)d_values);
}

void quotient_graph_run(h2b_ctx* ctx, const h2b_graph* g, uint32_t k, uint32_t ext_k, void* d_values) {
    check_domain(k, ext_k);
    GraphDev gd = graph_upload(ctx, g);
    H2B_LAUNCH(ctx, k_quotient_graph, ceil_div((size_t)1 << ext_k, 128), 128, 0, gd, ext_k, ext_k - k, (uint64_t*)d_values);
}

void lookup_fold_run(h2b_ctx* ctx, const h2b_graph* g, const void* d_z, const void* d_pin, const void* d_ptab, const void* d_l0,
                     const void* d_l_last, const void* d_l_active, uint32_t k, uint32_t ext_k, void* d_values) {
    check_domain(k, ext_k);
    GraphDev gd = graph_upload(ctx, g);
    H2B_LAUNCH(ctx, k_lookup_fold, ceil_div((size_t)1 << ext_k, 128), 128, 0, gd, (const uint64_t*)d_z, (const uint64_t*)d_pin,
               (const uint64_t*)d_ptab, (const uint64_t*)d_l0, (const uint64_t*)d_l_last, (const uint64_t*)d_l_active, ext_k, ext_k - k,
               (uint64_t*)d_values);
}

void permutation_fold_run(h2b_ctx* ctx, const void* const* d_z, size_t n_sets, const void* const* d_columns, const void* const* d_sigma,
                          size_t n_cols, size_t chunk_len, const void* d_l0, const void* d_l_last, const void* d_l_active,
                          const uint64_t beta[4], const uint64_t gamma[4], const uint64_t y[4], uint32_t blinding_factors, uint32_t k,
                          uint32_t ext_k, void* d_values) {
    check_domain(k, ext_k);
    if (n_sets == 0) return;  // `if !sets.is_empty()`
    H2B_REQUIRE(chunk_len >= 1 && n_cols >= 1 && n_sets == (n_cols + chunk_len - 1) / chunk_len, "permutation: n_sets != ceil(n_cols / chunk_len)");
    H2B_REQUIRE(n_cols < 65536, "permutation: too many columns");
    for (size_t i = 0; i < n_sets; i++) H2B_REQUIRE(d_z[i], "permutation: null product column");
    for (size_t i = 0; i < n_cols; i++) H2B_REQUIRE(d_columns[i] && d_sigma[i], "permutation: null column");
    auto al = [](size_t x) { return (x + 31) & ~(size_t)31; };
    const size_t o_z = 0, o_c = al(8 * n_sets), o_s = al(o_c + 8 * n_cols), o_w = al(o_s + 8 * n_cols), total = o_w + 32 * 29;
    std::vector<char> host(total, 0);
    memcpy(host.data() + o_z, d_z, 8 * n_sets);
    memcpy(host.data() + o_c, d_columns, 8 * n_cols);
    memcpy(host.data() + o_s, d_sigma, 8 * n_cols);
    for (uint32_t j = 0; j < ext_k; j++) memcpy(host.data() + o_w + 32 * j, FR_OMEGA[ext_k - j], 32);  // omega_ext^(2^j) = omega_{ext_k - j}
    char* d = (char*)ctx->get(WS_MISC, total);
    H2B_CUDA(cudaMemcpyAsync(d, host.data(), total, cudaMemcpyHostToDevice, ctx->stream));
    PermDev p;
    p.z = (const uint64_t* const*)(d + o_z);
    p.columns = (const uint64_t* const*)(d + o_c);
    p.sigma = (const uint64_t* const*)(d + o_s);
    p.omega_pow2 = (const uint64_t*)(d + o_w);
    p.n_sets = (u32)n_sets;
    p.n_cols = (u32)n_cols;
    p.chunk_len = (u32)chunk_len;
    p.last_rotation = -(int)(blinding_factors + 1);
    p.beta = fr_from(beta);
    p.gamma = fr_from(gamma);
    p.y = fr_from(y);
    p.zeta = fr_from(FR_ZETA_U64);
    p.delta = fr_from(FR_DELTA_U64);
    p.lo_bits = ext_k < 11 ? ext_k : 11;
    const size_t n_lo = (size_t)1 << p.lo_bits, n_hi = (size_t)1 << (ext_k - p.lo_bits);
    uint64_t* tables = (uint64_t*)ctx->get(WS_MISC2, 32 * (n_lo + n_hi));
    p.pow_lo = tables;
    p.pow_hi = tables + 4 * n_lo;
    H2B_LAUNCH(ctx, k_omega_tables, ceil_div(n_lo + n_hi, 256), 256, 0, p, ext_k, tables, tables + 4 * n_lo);
    H2B_LAUNCH(ctx, k_permutation_fold, ceil_div((size_t)1 << ext_k, 128), 128, 0, p, (const uint64_t*)d_l0, (const uint64_t*)d_l_last,
               (const uint64_t*)d_l_active, ext_k, ext_k - k, (uint64_t*)d_values);
}

}  // namespace h2b
