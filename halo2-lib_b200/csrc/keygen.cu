// keygen.cu — the permutation side of keygen_vk / keygen_pk for the circuit halo2-base builds, on the device: the constants
// columns, the copy calls in halo2-base's order, and sigma bit-exact to halo2's permutation Assembly (DESIGN.md §4.8, §4.11).
//
// Assembly::copy(a, b) returns when a and b are already in one cycle and otherwise swaps mapping[a] and mapping[b] (aux and
// sizes only answer "same cycle?").  So the final mapping is the product of the transpositions of the copies that joined
// two classes when they were made, in call order:  sigma = t_1 o t_2 o .. o t_F.  Those copies are the spanning forest
// Kruskal builds with weight = call index (unique: the weights are distinct), found here by Borůvka; sigma(x) is the walk
// from x that keeps crossing the largest forest edge below the last one crossed (t_F is applied first).
//   copies:  u32 cell-id pairs (c n + r, permutation column c in [c, c1.., a0.., l0.., i0..] order: F constants columns, then
//            a_j = F + j, l_t = F + A + t, i_m = F + A + L + m) in call order: break copies, lookup copies, advice equalities
//            sorted by (a, b), constant equalities sorted by (constant, cell) with distinct constant d in constants column
//            d mod F, row d div F, and then (assign_instances, after the region) the instance copies column by column;
//   forest:  hook-and-compress rounds: atomicMin of the incident edge index per component root; a root hooks onto the root
//            across its edge (of two roots that chose the same edge the lower stays a root); pointer jumping until flat;
//   walk:    2E darts (vertex, edge) sorted by lookup.cu's radix sort; a dart's successor is the dart before its twin at the
//            head vertex; pointer jumping to the terminal dart; sigma(x) = the head of the terminal of x's largest dart;
//   values:  sigma_c(r) = delta^c' omega^r', omega^r' from the domain's two-level power table.
// Every call here synchronises the stream and frees its scratch before it returns.
#include "h2b_internal.cuh"
#include "field.cuh"
#include "fr_domain_consts.inc"

namespace h2b {

static constexpr u32 NONE = 0xffffffffu;

// device scratch of one call (the call synchronises before it returns)
struct Scratch {
    void* p = nullptr;
    explicit Scratch(size_t bytes) { H2B_CUDA(cudaMalloc(&p, bytes ? bytes : 1)); }
    ~Scratch() { cudaFree(p); }
    template <class T>
    T* at(size_t byte_offset) const { return (T*)((char*)p + byte_offset); }
};
static size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

static u32 read_word(h2b_ctx* ctx, const u32* d) {
    u32* bounce = (u32*)ctx->get_pinned(0, 4096);
    H2B_CUDA(cudaMemcpyAsync(bounce, d, 4, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    return bounce[0];
}

// ------------------------------------------------------------------------------------------------------------ copies
struct Layout {
    const uint64_t* ends;  // ends[j] = start of gate column j + 1 in the virtual column (= bp_0 + .. + bp_j), j < nbp
    u32 nbp, n, F, A, L;  // F: the number of constants columns, the first F permutation columns
    uint64_t N;
};

// the cell assigned_advices records for virtual index p (< N): a break cell belongs to the column it ends
__device__ __forceinline__ u32 raw_cell(const Layout& y, uint64_t p) {
    u32 lo = 0, hi = y.nbp;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if (__ldg(y.ends + mid) >= p) hi = mid; else lo = mid + 1;
    }
    const uint64_t s = lo ? __ldg(y.ends + lo - 1) : 0;
    return (y.F + lo) * y.n + (u32)(p - s);
}

// the gate walk's layout: ends[j] = bp_0 + .. + bp_j uploaded to d_ends (nbp + 1 words, stream-ordered)
static Layout upload_layout(h2b_ctx* ctx, const char* who, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A,
                            size_t L, uint64_t* d_ends) {
    Layout y;
    y.nbp = (u32)nbp;
    y.n = (u32)1 << k;
    y.F = (u32)F;
    y.A = (u32)A;
    y.L = (u32)L;
    y.N = N;
    y.ends = d_ends;
    std::vector<uint64_t> ends(nbp + 1, 0);
    for (size_t j = 0, acc = 0; j < nbp; j++) {
        H2B_REQUIRE(break_points[j] < y.n, std::string(who) + ": a break point is >= 2^k");
        acc += break_points[j];
        ends[j] = acc;
    }
    H2B_CUDA(cudaMemcpyAsync(d_ends, ends.data(), 8 * (nbp + 1), cudaMemcpyHostToDevice, ctx->stream));
    return y;
}

// lookup copy i: raw(index[i]) ~ (l_{i mod L}, i / L); an index >= N sets bit 0 of *status
__global__ void __launch_bounds__(256) k_kg_lookup_edges(Layout y, const uint64_t* __restrict__ index, u32 m, uint2* __restrict__ edges,
                                                         u32* __restrict__ status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t p = __ldg(index + i);
    if (p >= y.N) atomicOr(status, 1u);
    edges[i] = make_uint2(p < y.N ? raw_cell(y, p) : 0, (y.F + y.A + i % y.L) * y.n + i / y.L);
}

// 256-bit sort keys: (a << 32 | b) of advice equality i; an index >= N sets bit 1 of *status
__global__ void __launch_bounds__(256) k_kg_pair_keys(const uint64_t* __restrict__ pairs, u32 m, uint64_t N, uint64_t* __restrict__ keys,
                                                      u32* __restrict__ status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t a = __ldg(pairs + 2 * (size_t)i), b = __ldg(pairs + 2 * (size_t)i + 1);
    if (a >= N || b >= N) atomicOr(status, 2u);
    const ulonglong4 key = {a < N && b < N ? (a << 32 | b) : 0, 0, 0, 0};
    reinterpret_cast<ulonglong4*>(keys)[i] = key;
}

// advice equality i of the sorted order: raw(a) ~ raw(b)
__global__ void __launch_bounds__(256) k_kg_pair_edges(Layout y, const uint64_t* __restrict__ keys, const u32* __restrict__ order, u32 m,
                                                       uint2* __restrict__ edges) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t key = __ldg(keys + 4 * (size_t)__ldg(order + i));
    edges[i] = make_uint2(raw_cell(y, key >> 32), raw_cell(y, key & 0xffffffffull));
}

// keys of the constant equalities: the cell index, then (second sort) the canonical constant; an index >= N sets bit 1
__global__ void __launch_bounds__(256) k_kg_const_keys(const uint64_t* __restrict__ consts, const uint64_t* __restrict__ index, u32 m, uint64_t N,
                                                       uint64_t* __restrict__ index_keys, uint64_t* __restrict__ const_keys, u32* __restrict__ status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t p = __ldg(index + i);
    if (p >= N) atomicOr(status, 2u);
    const ulonglong4 ik = {p < N ? p : 0, 0, 0, 0};
    reinterpret_cast<ulonglong4*>(index_keys)[i] = ik;
    const Fr v = Fr::load_nc(consts + 4 * (size_t)i).from_mont();
    const ulonglong4 ck = {(uint64_t)v.l[0] | (uint64_t)v.l[1] << 32, (uint64_t)v.l[2] | (uint64_t)v.l[3] << 32,
                           (uint64_t)v.l[4] | (uint64_t)v.l[5] << 32, (uint64_t)v.l[6] | (uint64_t)v.l[7] << 32};
    reinterpret_cast<ulonglong4*>(const_keys)[i] = ck;
}

__global__ void k_kg_add_word(const u32* __restrict__ a, u32* __restrict__ acc) { *acc += *a; }

// heads[i] = 1 where the i-th constant of the sorted order differs from the one before it
__global__ void __launch_bounds__(256) k_kg_const_heads(const uint64_t* __restrict__ const_keys, const u32* __restrict__ order, u32 m,
                                                        u32* __restrict__ heads) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    bool head = i == 0;
    if (!head) {
        const ulonglong4 a = reinterpret_cast<const ulonglong4*>(const_keys)[__ldg(order + i)];
        const ulonglong4 b = reinterpret_cast<const ulonglong4*>(const_keys)[__ldg(order + i - 1)];
        head = a.x != b.x || a.y != b.y || a.z != b.z || a.w != b.w;
    }
    heads[i] = head ? 1u : 0u;
}

// constant equality i of the sorted order: the cell of its constant ~ raw(cell).  Distinct constant d (the rank of its run's
// head) goes left to right, then top to bottom: constants column d mod F, row d div F, cell id (d mod F) n + d div F, which is
// also its offset in the F x n block c_block.  Each head places its constant there; a rank >= F n is not written (F = 0: none
// is; the caller raises NotEnoughRowsAvailable, or the index-out-of-bounds panic when F = 0)
__global__ void __launch_bounds__(256) k_kg_const_edges(Layout y, const uint64_t* __restrict__ consts, const uint64_t* __restrict__ index,
                                                        const u32* __restrict__ order, const u32* __restrict__ heads, const u32* __restrict__ rows,
                                                        u32 m, uint64_t* __restrict__ c_block, uint2* __restrict__ edges) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const u32 src = __ldg(order + i), d = __ldg(rows + i) + __ldg(heads + i) - 1;
    const uint64_t p = __ldg(index + src);
    u32 cell = 0;
    if (d < y.F * y.n) {
        cell = (d % y.F) * y.n + d / y.F;
        if (__ldg(heads + i)) Fr::load_nc(consts + 4 * (size_t)src).store(c_block + 4 * (size_t)cell);
    }
    edges[i] = make_uint2(cell, p < y.N ? raw_cell(y, p) : 0);
}

void keygen_copies_run(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                       const uint64_t* d_lookup_index, size_t n_lookup, const uint64_t* d_pairs, size_t M, const void* d_consts,
                       const uint64_t* d_const_index, size_t Mc, void* d_c, void* d_edges, uint32_t* status) {
    H2B_REQUIRE(k >= 3 && k <= 28, "keygen_copies: k out of range (3..28)");
    const size_t n = (size_t)1 << k;
    H2B_REQUIRE(A >= 1 && nbp < A, "keygen_copies: need A >= 1 gate columns and fewer break points than that");
    H2B_REQUIRE(F < NONE && (F + A + L) * n < NONE, "keygen_copies: the permutation columns hold more than 2^32 - 1 cells");
    H2B_REQUIRE(N < ((size_t)1 << 32) && n_lookup < ((size_t)1 << 31) && M < ((size_t)1 << 31) && Mc < ((size_t)1 << 31),
                "keygen_copies: at most 2^32 - 1 cells and 2^31 - 1 copies of each kind");
    H2B_REQUIRE(L || n_lookup == 0, "keygen_copies: lookup copies need lookup-advice columns");
    const u32 m = (u32)std::max(M, Mc);
    const int ctas = sort_column_ctas(ctx, std::max<u32>(m, 1));
    // scratch: ends | keys (32 m) | second keys (32 m) | order (4 m) | order2 (4 m) | heads (4 m) | rows (4 m) | sort | scan
    const size_t o_keys = al(8 * (nbp + 1)), o_keys2 = o_keys + al(32 * (size_t)m), o_ord = o_keys2 + al(32 * (size_t)m),
                 o_ord2 = o_ord + al(4 * (size_t)m), o_heads = o_ord2 + al(4 * (size_t)m), o_rows = o_heads + al(4 * (size_t)m),
                 o_sort = o_rows + al(4 * (size_t)m), o_scan = o_sort + al(sort_keys_scratch(m, ctas));
    Scratch s(o_scan + al(exclusive_scan_scratch(m)));
    const Layout y = upload_layout(ctx, "keygen_copies", N, break_points, nbp, k, F, A, L, s.at<uint64_t>(0));
    std::vector<uint32_t> brk(2 * nbp);
    for (size_t j = 0; j < nbp; j++) {
        brk[2 * j] = (u32)((F + 1 + j) * n);                    // (a_{j+1}, 0)
        brk[2 * j + 1] = (u32)((F + j) * n + break_points[j]);  // (a_j, bp_j)
    }
    uint2* edges = (uint2*)d_edges;
    H2B_CUDA(cudaMemsetAsync(status, 0, 8, ctx->stream));
    if (F) H2B_CUDA(cudaMemsetAsync(d_c, 0, 32 * F * n, ctx->stream));
    if (nbp) H2B_CUDA(cudaMemcpyAsync(edges, brk.data(), 8 * nbp, cudaMemcpyHostToDevice, ctx->stream));
    edges += nbp;
    if (n_lookup) H2B_LAUNCH(ctx, k_kg_lookup_edges, ceil_div(n_lookup, 256), 256, 0, y, d_lookup_index, (u32)n_lookup, edges, status);
    edges += n_lookup;
    uint64_t* keys = s.at<uint64_t>(o_keys);
    uint64_t* keys2 = s.at<uint64_t>(o_keys2);
    u32* order = s.at<u32>(o_ord);
    u32* order2 = s.at<u32>(o_ord2);
    if (M) {
        H2B_LAUNCH(ctx, k_kg_pair_keys, ceil_div(M, 256), 256, 0, d_pairs, (u32)M, (uint64_t)N, keys, status);
        sort_keys(ctx, keys, (u32)M, nullptr, order, s.at<char>(o_sort), ctas);
        H2B_LAUNCH(ctx, k_kg_pair_edges, ceil_div(M, 256), 256, 0, y, (const uint64_t*)keys, (const u32*)order, (u32)M, edges);
    }
    edges += M;
    if (Mc) {
        u32* heads = s.at<u32>(o_heads);
        u32* rows = s.at<u32>(o_rows);
        H2B_LAUNCH(ctx, k_kg_const_keys, ceil_div(Mc, 256), 256, 0, (const uint64_t*)d_consts, d_const_index, (u32)Mc, (uint64_t)N, keys, keys2, status);
        sort_keys(ctx, keys, (u32)Mc, nullptr, order, s.at<char>(o_sort), ctas);         // by cell
        sort_keys(ctx, keys2, (u32)Mc, order, order2, s.at<char>(o_sort), ctas);         // then stably by constant
        H2B_LAUNCH(ctx, k_kg_const_heads, ceil_div(Mc, 256), 256, 0, (const uint64_t*)keys2, (const u32*)order2, (u32)Mc, heads);
        exclusive_scan(ctx, heads, (u32)Mc, rows, s.at<char>(o_scan));
        H2B_LAUNCH(ctx, k_kg_const_edges, ceil_div(Mc, 256), 256, 0, y, (const uint64_t*)d_consts, d_const_index, (const u32*)order2,
                   (const u32*)heads, (const u32*)rows, (u32)Mc, (uint64_t*)d_c, edges);
        // status[1] = distinct constants = the last row + its head flag
        u32* last = status + 1;
        H2B_CUDA(cudaMemcpyAsync(last, rows + Mc - 1, 4, cudaMemcpyDeviceToDevice, ctx->stream));
        H2B_LAUNCH(ctx, k_kg_add_word, 1, 1, 0, (const u32*)(heads + Mc - 1), last);
    }
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
}

// instance copy r of column `col` (assign_instances): raw(index[r]) ~ (i_col, r).  *status (this column's word): bit 0 an index
// >= N at a row <= usable (halo2-base's expect runs before the copy of the same row), bit 1 a row >= usable (Assembly::copy
// fails there); such copies are written as the no-op (0, 0)
__global__ void __launch_bounds__(256) k_kg_instance_edges(Layout y, const uint64_t* __restrict__ index, u32 m, u32 col, u32 usable,
                                                           uint2* __restrict__ edges, u32* __restrict__ status) {
    const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= m) return;
    const uint64_t p = __ldg(index + r);
    if (p >= y.N && r <= usable) atomicOr(status, 1u);
    if (r >= usable) atomicOr(status, 2u);
    const bool ok = p < y.N && r < usable;
    edges[r] = ok ? make_uint2(raw_cell(y, p), (y.F + y.A + y.L + col) * y.n + r) : make_uint2(0, 0);
}

void keygen_instance_edges_run(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                               size_t usable, size_t I, const size_t* n_index, const uint64_t* d_index, void* d_edges, uint32_t* status) {
    H2B_REQUIRE(k >= 3 && k <= 28, "keygen_instance_edges: k out of range (3..28)");
    const size_t n = (size_t)1 << k;
    H2B_REQUIRE(A >= 1 && nbp < A && usable <= n, "keygen_instance_edges: need A >= 1 gate columns, fewer break points and usable <= 2^k");
    H2B_REQUIRE(F < NONE && I < NONE && (F + A + L + I) * n < NONE, "keygen_instance_edges: the permutation columns hold more than 2^32 - 1 cells");
    H2B_REQUIRE(N < ((size_t)1 << 32), "keygen_instance_edges: at most 2^32 - 1 cells");
    Scratch s(8 * (nbp + 1));
    const Layout y = upload_layout(ctx, "keygen_instance_edges", N, break_points, nbp, k, F, A, L, s.at<uint64_t>(0));
    if (I) H2B_CUDA(cudaMemsetAsync(status, 0, 4 * I, ctx->stream));
    uint2* edges = (uint2*)d_edges;
    for (size_t col = 0; col < I; col++) {
        H2B_REQUIRE(n_index[col] < ((size_t)1 << 31), "keygen_instance_edges: at most 2^31 - 1 cells per instance column");
        if (n_index[col])
            H2B_LAUNCH(ctx, k_kg_instance_edges, ceil_div(n_index[col], 256), 256, 0, y, d_index, (u32)n_index[col], (u32)col, (u32)usable, edges,
                       status + col);
        d_index += n_index[col];
        edges += n_index[col];
    }
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
}

// ------------------------------------------------------------------------------------------------------------ forest
__global__ void __launch_bounds__(256) k_kg_iota(u32* __restrict__ a, u32 n) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = i;
}

// best[root] = the smallest index of an edge joining the root's component to another one (parent is flat); a cell id >= V
// sets *bad
__global__ void __launch_bounds__(256) k_kg_min_edge(const uint2* __restrict__ edges, u32 E, u32 V, const u32* __restrict__ parent,
                                                     u32* __restrict__ best, u32* __restrict__ bad) {
    const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const uint2 ed = edges[e];
    if (ed.x >= V || ed.y >= V) {
        atomicOr(bad, 1u);
        return;
    }
    const u32 ra = __ldg(parent + ed.x), rb = __ldg(parent + ed.y);
    if (ra == rb) return;
    atomicMin(best + ra, e);
    atomicMin(best + rb, e);
}

// every root with a chosen edge marks it as a forest edge and hooks onto the root across it (reads parent, writes next); of
// two roots that chose the same edge, the lower one stays a root
__global__ void __launch_bounds__(256) k_kg_hook(const uint2* __restrict__ edges, u32 V, const u32* __restrict__ parent, const u32* __restrict__ best,
                                                 u32* __restrict__ next, uint8_t* __restrict__ forest, u32* __restrict__ hooked) {
    const u32 v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V || __ldg(parent + v) != v) return;
    const u32 e = __ldg(best + v);
    if (e == NONE) return;
    const uint2 ed = edges[e];
    const u32 ra = __ldg(parent + ed.x), rb = __ldg(parent + ed.y), other = ra == v ? rb : ra;
    forest[e] = 1;
    if (__ldg(best + other) == e && v < other) return;
    next[v] = other;
    *hooked = 1;  // every writer stores the same word
}

// pointer jumping: p[v] <- p[p[v]] up to 4 times; *changed when v's pointer does not reach a fixed point yet
__global__ void __launch_bounds__(256) k_kg_jump(u32* __restrict__ p, u32 V, u32* __restrict__ changed) {
    const u32 v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    u32 x = p[v], y = p[x];
    if (x == y) return;
    for (int it = 0; it < 4 && x != y; it++) {
        x = y;
        y = p[x];
    }
    p[v] = x;
    if (x != y) atomicOr(changed, 1u);
}

static void flatten(h2b_ctx* ctx, u32* p, u32 V, u32* flag) {
    for (;;) {
        H2B_CUDA(cudaMemsetAsync(flag, 0, 4, ctx->stream));
        H2B_LAUNCH(ctx, k_kg_jump, ceil_div(V, 256), 256, 0, p, V, flag);
        if (!read_word(ctx, flag)) return;
    }
}

// -------------------------------------------------------------------------------------------------------------- walk
// dart d of edge d / 2: at the edge's first (d even) or second cell; key = vertex << 32 | edge, or all ones off the forest
__global__ void __launch_bounds__(256) k_kg_dart_keys(const uint2* __restrict__ edges, const uint8_t* __restrict__ forest, u32 D,
                                                      uint64_t* __restrict__ keys) {
    const u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    const u32 e = d >> 1;
    const uint2 ed = edges[e];
    const ulonglong4 key = {forest[e] ? ((uint64_t)((d & 1) ? ed.y : ed.x) << 32 | e) : ~0ull, 0, 0, 0};
    reinterpret_cast<ulonglong4*>(keys)[d] = key;
}

__global__ void __launch_bounds__(256) k_kg_dart_pos(const u32* __restrict__ order, u32 D, u32* __restrict__ pos) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < D) pos[order[i]] = i;
}

__device__ __forceinline__ uint64_t dart_key(const uint64_t* keys, u32 d) { return __ldg(keys + 4 * (size_t)d); }

// in sorted positions: head[i] = the vertex dart i leads to; nxt[i] = the dart taken there (the one before its twin, the
// largest smaller edge at that vertex) or i itself when the walk ends
__global__ void __launch_bounds__(256) k_kg_dart_next(const uint64_t* __restrict__ keys, const u32* __restrict__ order, const u32* __restrict__ pos,
                                                      u32 D, u32* __restrict__ nxt, u32* __restrict__ head) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D) return;
    const u32 d = __ldg(order + i);
    nxt[i] = i;
    if (dart_key(keys, d) == ~0ull) return;
    const u32 twin = d ^ 1u, j = __ldg(pos + twin), w = (u32)(dart_key(keys, twin) >> 32);
    head[i] = w;
    if (j > 0 && (u32)(dart_key(keys, __ldg(order + j - 1)) >> 32) == w) nxt[i] = j - 1;
}

// map[x] = the head of the terminal dart of x's largest dart
__global__ void __launch_bounds__(256) k_kg_dart_map(const uint64_t* __restrict__ keys, const u32* __restrict__ order, const u32* __restrict__ nxt,
                                                     const u32* __restrict__ head, u32 D, u32* __restrict__ map) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D) return;
    const uint64_t key = dart_key(keys, __ldg(order + i));
    if (key == ~0ull) return;
    if (i + 1 < D && dart_key(keys, __ldg(order + i + 1)) >> 32 == key >> 32) return;
    map[key >> 32] = __ldg(head + __ldg(nxt + i));
}

void keygen_sigma_map_run(h2b_ctx* ctx, const void* d_edges, size_t E, size_t n_cols, uint32_t k, void* d_map) {
    H2B_REQUIRE(k >= 1 && k <= 28, "keygen_sigma_map: k out of range (1..28)");
    H2B_REQUIRE(n_cols >= 1 && (n_cols << k) < NONE, "keygen_sigma_map: the permutation columns hold more than 2^32 - 1 cells");
    H2B_REQUIRE(E < ((size_t)1 << 31), "keygen_sigma_map: at most 2^31 - 1 copies");
    const u32 V = (u32)(n_cols << k), D = (u32)(2 * E);
    u32* map = (u32*)d_map;
    H2B_LAUNCH(ctx, k_kg_iota, ceil_div(V, 256), 256, 0, map, V);
    if (E == 0) {
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
        return;
    }
    const uint2* edges = (const uint2*)d_edges;
    const int ctas = sort_column_ctas(ctx, D);
    // scratch: flags (16) | parent, next, best (4 V each) | forest (E) | dart keys (32 D) | order, pos, nxt, head (4 D each) | sort
    const size_t o_par = 256, o_next = o_par + al(4 * (size_t)V), o_best = o_next + al(4 * (size_t)V), o_forest = o_best + al(4 * (size_t)V),
                 o_keys = o_forest + al(E), o_ord = o_keys + al(32 * (size_t)D), o_pos = o_ord + al(4 * (size_t)D), o_nxt = o_pos + al(4 * (size_t)D),
                 o_head = o_nxt + al(4 * (size_t)D), o_sort = o_head + al(4 * (size_t)D);
    Scratch s(o_sort + al(sort_keys_scratch(D, ctas)));
    u32* flag = s.at<u32>(0);
    u32 *parent = s.at<u32>(o_par), *next = s.at<u32>(o_next), *best = s.at<u32>(o_best);
    uint8_t* forest = s.at<uint8_t>(o_forest);
    H2B_LAUNCH(ctx, k_kg_iota, ceil_div(V, 256), 256, 0, parent, V);
    H2B_CUDA(cudaMemsetAsync(forest, 0, E, ctx->stream));
    for (int round = 0;; round++) {
        H2B_CUDA(cudaMemsetAsync(flag, 0, 8, ctx->stream));
        H2B_CUDA(cudaMemsetAsync(best, 0xff, 4 * (size_t)V, ctx->stream));
        H2B_LAUNCH(ctx, k_kg_min_edge, ceil_div(E, 256), 256, 0, edges, (u32)E, V, (const u32*)parent, best, flag + 1);
        H2B_CUDA(cudaMemcpyAsync(next, parent, 4 * (size_t)V, cudaMemcpyDeviceToDevice, ctx->stream));
        H2B_LAUNCH(ctx, k_kg_hook, ceil_div(V, 256), 256, 0, edges, V, (const u32*)parent, (const u32*)best, next, forest, flag);
        if (round == 0 && read_word(ctx, flag + 1)) throw StatusError{H2B_ERR_ARG, "keygen_sigma_map: a copy names a cell outside the permutation columns"};
        if (!read_word(ctx, flag)) break;
        flatten(ctx, next, V, flag + 2);
        std::swap(parent, next);
    }
    uint64_t* keys = s.at<uint64_t>(o_keys);
    u32 *order = s.at<u32>(o_ord), *pos = s.at<u32>(o_pos), *nxt = s.at<u32>(o_nxt), *head = s.at<u32>(o_head);
    H2B_LAUNCH(ctx, k_kg_dart_keys, ceil_div(D, 256), 256, 0, edges, (const uint8_t*)forest, D, keys);
    sort_keys(ctx, keys, D, nullptr, order, s.at<char>(o_sort), ctas);
    H2B_LAUNCH(ctx, k_kg_dart_pos, ceil_div(D, 256), 256, 0, (const u32*)order, D, pos);
    H2B_LAUNCH(ctx, k_kg_dart_next, ceil_div(D, 256), 256, 0, (const uint64_t*)keys, (const u32*)order, (const u32*)pos, D, nxt, head);
    flatten(ctx, nxt, D, flag + 2);
    H2B_LAUNCH(ctx, k_kg_dart_map, ceil_div(D, 256), 256, 0, (const uint64_t*)keys, (const u32*)order, (const u32*)nxt, (const u32*)head, D, map);
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
}

// ------------------------------------------------------------------------------------------------------------ values
__global__ void k_kg_delta_pows(Fr delta, u32 n_cols, uint64_t* __restrict__ out) {
    Fr x = Fr::one();
    for (u32 c = 0; c < n_cols; c++, x = x * delta) x.store(out + 4 * (size_t)c);
}

// sigma[x] = delta^c' omega^r' for map[x] = c' 2^k + r'
__global__ void __launch_bounds__(256) k_kg_sigma_values(const u32* __restrict__ map, u32 V, u32 k, const uint64_t* __restrict__ dpow,
                                                         const uint64_t* __restrict__ lo, const uint64_t* __restrict__ hi, u32 h,
                                                         uint64_t* __restrict__ sigma) {
    const u32 x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= V) return;
    const u32 m = __ldg(map + x), c = m >> k, r = m & ((1u << k) - 1);
    Fr v = Fr::load_nc(lo + 4 * (size_t)(r & ((1u << h) - 1)));
    if (r >> h) v = v * Fr::load_nc(hi + 4 * (size_t)(r >> h));
    if (c) v = v * Fr::load_nc(dpow + 4 * (size_t)c);
    v.store(sigma + 4 * (size_t)x);
}

void keygen_sigma_values_run(h2b_ctx* ctx, const void* d_map, size_t n_cols, uint32_t k, void* d_sigma) {
    H2B_REQUIRE(k >= 1 && k <= 28, "keygen_sigma_values: k out of range (1..28)");
    H2B_REQUIRE(n_cols >= 1 && (n_cols << k) < NONE, "keygen_sigma_values: the permutation columns hold more than 2^32 - 1 cells");
    const void *lo, *hi;
    int h;
    domain_power_tables(ctx, k, &lo, &hi, &h);
    Scratch s(32 * n_cols);
    Fr delta;
    memcpy(&delta, FR_DELTA_U64, sizeof(Fr));
    H2B_LAUNCH(ctx, k_kg_delta_pows, 1, 1, 0, delta, (u32)n_cols, s.at<uint64_t>(0));
    const u32 V = (u32)(n_cols << k);
    H2B_LAUNCH(ctx, k_kg_sigma_values, ceil_div(V, 256), 256, 0, (const u32*)d_map, V, k, (const uint64_t*)s.p, (const uint64_t*)lo,
               (const uint64_t*)hi, (u32)h, (uint64_t*)d_sigma);
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
}

}  // namespace h2b
