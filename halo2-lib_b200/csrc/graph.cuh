// graph.cuh — the device side of the h2b_graph interpreter (GraphEvaluator programs, include/h2b200.h), shared by the
// quotient kernels (quotient.cu: one row of the extended coset per thread) and the constraint check (check.cu: one row of
// the 2^k domain per thread, rotation shift 0).
#pragma once
#include "h2b_internal.cuh"
#include "field.cuh"

namespace h2b {

static constexpr u32 CALC_NOP = 8;  // internal: see graph_upload

struct GraphDev {
    const u32* program;
    u32 n_calc, result;
    const uint64_t* constants;
    const int32_t* rotations;
    const uint64_t* const* fixed;
    const uint64_t* const* advice;
    const uint64_t* const* instance;
    const uint64_t* challenges;
    Fr beta, gamma, theta, y;
};

// validates the program, resolves its Stores and copies program + tables into one device blob (workspace WS_MISC)
GraphDev graph_upload(h2b_ctx* ctx, const h2b_graph* g);

__device__ __forceinline__ size_t rot_idx(size_t idx, int rot, u32 rshift, size_t mask) {
    return (size_t)((long long)idx + (long long)rot * ((long long)1 << rshift)) & mask;  // get_rotation_idx
}

__device__ __forceinline__ Fr graph_fetch(const GraphDev& g, u32 src, size_t idx, size_t mask, u32 rshift, const Fr& prev,
                                       const Fr* inter) {
    const u32 kind = src & 15u, index = (src >> 4) & 0xffffu, slot = src >> 20;
    switch (kind) {
        case H2B_SRC_CONSTANT: return Fr::load_nc(g.constants + 4 * (size_t)index);
        case H2B_SRC_INTERMEDIATE: return inter[index];
        case H2B_SRC_FIXED: return Fr::load_nc(g.fixed[index] + 4 * rot_idx(idx, g.rotations[slot], rshift, mask));
        case H2B_SRC_ADVICE: return Fr::load_nc(g.advice[index] + 4 * rot_idx(idx, g.rotations[slot], rshift, mask));
        case H2B_SRC_INSTANCE: return Fr::load_nc(g.instance[index] + 4 * rot_idx(idx, g.rotations[slot], rshift, mask));
        case H2B_SRC_CHALLENGE: return Fr::load_nc(g.challenges + 4 * (size_t)index);
        case H2B_SRC_BETA: return g.beta;
        case H2B_SRC_GAMMA: return g.gamma;
        case H2B_SRC_THETA: return g.theta;
        case H2B_SRC_Y: return g.y;
        default: return prev;  // H2B_SRC_PREVIOUS (the host validated the program)
    }
}

// runs the straight-line program for row idx; returns the value of g.result
__device__ __forceinline__ Fr graph_eval(const GraphDev& g, size_t idx, size_t mask, u32 rshift, const Fr& prev, Fr* inter) {
    const u32* pc = g.program;
#pragma unroll 1
    for (u32 t = 0; t < g.n_calc; t++) {
        const u32 op = __ldg(pc++);
        if (op == CALC_NOP) continue;  // a Store the host resolved into its users
        Fr r;
        if (op == H2B_CALC_HORNER) {
            r = graph_fetch(g, __ldg(pc), idx, mask, rshift, prev, inter);
            const Fr f = graph_fetch(g, __ldg(pc + 1), idx, mask, rshift, prev, inter);
            const u32 np = __ldg(pc + 2);
            pc += 3;
#pragma unroll 1
            for (u32 j = 0; j < np; j++) r = r * f + graph_fetch(g, __ldg(pc++), idx, mask, rshift, prev, inter);
        } else {
            const Fr a = graph_fetch(g, __ldg(pc++), idx, mask, rshift, prev, inter);
            if (op <= H2B_CALC_MUL) {
                const Fr b = graph_fetch(g, __ldg(pc++), idx, mask, rshift, prev, inter);
                r = (op == H2B_CALC_ADD) ? a + b : (op == H2B_CALC_SUB) ? a - b : a * b;
            } else if (op == H2B_CALC_SQUARE) r = a.sqr();
            else if (op == H2B_CALC_DOUBLE) r = a.dbl();
            else if (op == H2B_CALC_NEGATE) r = a.neg();
            else r = a;  // H2B_CALC_STORE
        }
        inter[t] = r;
    }
    return graph_fetch(g, g.result, idx, mask, rshift, prev, inter);
}

}  // namespace h2b
