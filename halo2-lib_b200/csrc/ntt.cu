// ntt.cu — number-theoretic transform over BN254 Fr for sm_90a.
//
// Replaces halo2-axiom 0.5.3 `arithmetic::best_fft(a, omega, log_n)` and the EvaluationDomain wrappers
// lagrange_to_coeff / coeff_to_lagrange / coeff_to_extended / extended_to_coeff that create_proof calls per
// column (SURVEY.md §3.3 steps 3-6, §8 a3, Appendix B).  Contract: natural order in, natural order out,
// out[i] = sum_j a[j] * omega^(i*j).
//
// Decomposition: log_n = r_1 + ... + r_p (p <= 3, r_t <= 11).  Pass t transforms digit t of the index
// (decimation in frequency) for a tile of 2^r_t rows x CW adjacent columns held in shared memory (two
// 128-bit planes per element, conflict-free for unit-stride lanes), multiplies by the inter-pass twiddle
// omega_t^(i_t * j') (one precomputed table entry per in-place address, built once per domain from a two-level
// power table of omega, with 2^-k folded in for inverse transforms), and writes in place; the last pass
// writes through the digit-reversal so the result is in natural order with >= 64-byte contiguous stores.
// Every pass reads and writes each element once: 64 B of HBM traffic per element per pass.
// Coset scaling (zeta^(i mod 3)) and zero padding are fused into the first pass, zeta^-(i mod 3) into the last.
#include "h2b_internal.cuh"
#include "field.cuh"
#include "fr_domain_consts.inc"

namespace h2b {

static constexpr int NTT_THREADS = 256;   // upper bound; small tiles run with TILE / 4 threads (one radix-4 group each)
static constexpr int NTT_TILE_LOG = 11;  // largest tile: 2^11 elements * 32 B = 64 KB of shared memory
static constexpr int NTT_SMEM_MAX = 227 * 1024;  // opt-in limit of dynamic shared memory per CTA on sm_90
static constexpr int NTT_MAX_R = 11;  // one column of the largest digit = 2^11 * 32 B = the whole 64 KB tile

// Fr::ZETA and ZETA^2 in Montgomery form (halo2curves bn256::Fr::ZETA; SURVEY.md §8c); the same values are
// emitted as FR_ZETA_U32 by tools/gen_domain_consts.py
__device__ __forceinline__ Fr fr_zeta(int pw) {  // pw in {1,2}
    Fr z;
    if (pw == 1) {
        z.l[0] = 0x55fcd653u; z.l[1] = 0x0363f299u; z.l[2] = 0x5fc1e200u; z.l[3] = 0x73e7950bu;
        z.l[4] = 0x576d9d24u; z.l[5] = 0xc5fce83eu; z.l[6] = 0xa1c3a4d4u; z.l[7] = 0x059c805du;
    } else {
        z.l[0] = 0x4a0329b3u; z.l[1] = 0x93e7cedeu; z.l[2] = 0x7a96c167u; z.l[3] = 0x7d4fdca7u;
        z.l[4] = 0xb19a750au; z.l[5] = 0x8be4ba08u; z.l[6] = 0xa5661c25u; z.l[7] = 0x1cbd5653u;
    }
    return z;
}

struct NttPlan {
    uint32_t log_n = 0;
    int npass = 0;
    int r[3] = {0, 0, 0};
    int h = 0;                 // tw_lo has 2^h entries, tw_hi 2^(log_n - h)
    Fr* tw_lo = nullptr;       // omega^i
    Fr* tw_hi = nullptr;       // omega^(i << h)
    Fr* wtab[3] = {nullptr, nullptr, nullptr};  // per pass: rho_t^e, e < 2^(r_t - 1), rho_t = omega^(n / 2^r_t)
    Fr* n_inv = nullptr;       // 2^-log_n
    Fr* tw_full[2] = {nullptr, nullptr};  // per non-last pass: the inter-pass twiddle of every in-place address
                                          // (times 2^-log_n in the first one when the plan scales)
    int scaled = 0;
    void* block = nullptr;
    void* block2 = nullptr;
    bool domain_root = false;  // omega is the 2^log_n domain root or its inverse (kept for the context's lifetime)
    uint64_t seq = 0;          // creation order, for the eviction of plans built for arbitrary roots
};
static constexpr size_t NTT_MAX_ADHOC_PLANS = 4;  // best_fft with arbitrary roots: bounded cache (a plan can hold n x 32 B per pass)

// out[i] = omega^(i * mult)
__global__ void k_pow_table(Fr omega, uint64_t mult, u32 count, Fr* __restrict__ out) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint64_t e = (uint64_t)i * mult;
    Fr acc = Fr::one(), base = omega;
    while (e) {
        if (e & 1) acc = acc * base;
        base = base.sqr();
        e >>= 1;
    }
    acc.store(out + i);
}
__global__ void k_n_inv(u32 log_n, Fr* out) {
    Fr two = Fr::one() + Fr::one(), acc = Fr::one();
    for (u32 i = 0; i < log_n; i++) acc = acc * two;
    acc.inv_bgcd().store(out);
}

// tw_full[g] = omega_t^(row * j') (times n_inv when given) for every in-place address g of a non-last pass
__global__ void k_tw_full(const Fr* __restrict__ tw_lo, const Fr* __restrict__ tw_hi, int h, int log_n, int r, int logM,
                          int tw_shift, const Fr* __restrict__ n_inv, Fr* __restrict__ out) {
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ((size_t)1 << log_n)) return;
    u32 jp = (u32)(g & (((size_t)1 << logM) - 1));
    u32 row = (u32)((g >> logM) & ((1u << r) - 1));
    uint64_t ex = ((uint64_t)row * jp) << tw_shift;
    Fr t = Fr::load_nc(tw_lo + (ex & ((1ull << h) - 1)));
    uint64_t eh = ex >> h;
    if (eh) t = t * Fr::load_nc(tw_hi + eh);
    if (n_inv) t = t * Fr::load_nc(n_inv);
    t.store(out + g);
}

struct PassArgs {
    const Fr* in;
    Fr* out;
    u32 n_in;        // elements present in `in` (first pass; beyond -> zero)
    int log_n, r, logM, cw_log;
    int first, last;
    int logN1, logBrest;   // last pass: natural index = i1 + N1 * (rest + Brest * row)
    const Fr* wtab;
    const Fr* n_inv; // non-null: scale by 2^-log_n in the last pass
    const Fr* tw_full; // non-last passes: precomputed twiddle per in-place address
    int coset;       // 1: in[i] *= zeta^(i mod 3) on load (first pass); 2: out[i] *= zeta^-(i mod 3) on store (last)
};

struct SmemFr {  // two 128-bit planes
    uint4* lo;
    uint4* hi;
    __device__ __forceinline__ Fr ld(u32 i) const {
        uint4 a = lo[i], b = hi[i];
        Fr r;
        r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
        r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
        return r;
    }
    __device__ __forceinline__ void st(u32 i, const Fr& v) const {
        lo[i] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
        hi[i] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    }
};

template <bool LAST>
__global__ void __launch_bounds__(NTT_THREADS, 3) k_ntt_pass(PassArgs a) {
    extern __shared__ uint4 smem_raw[];
    const int r = a.r, cwl = a.cw_log;
    const u32 R = 1u << r, CW = 1u << cwl, TILE = R << cwl;
    SmemFr sm{smem_raw, smem_raw + TILE};
    const u32 col0 = blockIdx.x << cwl;
    const int tid = threadIdx.x;
    const u32 NT = blockDim.x;

    // shared index of (row, c): the last pass keeps columns contiguous (its global rows are contiguous)
    auto sidx = [&](u32 row, u32 c) -> u32 { return LAST ? (c << r) + row : (row << cwl) + c; };
    // global address (in-place digit layout) of (row, col)
    auto gaddr = [&](u32 row, u32 col) -> size_t {
        if (LAST) {
            u32 i1 = col & ((1u << a.logN1) - 1), rest = col >> a.logN1;
            size_t b = ((size_t)i1 << a.logBrest) + rest;
            return (b << r) + row;
        } else {
            size_t b = col >> a.logM;
            u32 jp = col & ((1u << a.logM) - 1);
            return (b << (r + a.logM)) + ((size_t)row << a.logM) + jp;
        }
    };

    // ---- load
    for (u32 e = tid; e < TILE; e += NT) {
        u32 row, c;
        if (LAST) { row = e & (R - 1); c = e >> r; } else { c = e & (CW - 1); row = e >> cwl; }
        size_t g = gaddr(row, col0 + c);
        Fr v = Fr::zero();
        if (g < a.n_in) {
            v = Fr::load(a.in + g);
            if (a.coset == 1 && a.first) {
                u32 m = (u32)(g % 3);
                if (m) v = v * fr_zeta((int)m);
            }
        }
        sm.st(sidx(row, c), v);
    }
    __syncthreads();

    // ---- r radix-2 DIF stages inside the tile, two at a time: a thread takes the 4 elements u, u+q, u+2q, u+3q
    // (q = quarter of the current block), does the stage-s butterflies (u, u+2q), (u+q, u+3q) and the stage-(s+1)
    // butterflies (u, u+q), (u+2q, u+3q) in registers: half the shared-memory round trips and barriers.
    const u32 NBF = TILE >> 1;
    int s = 0;
    for (; s + 1 < r; s += 2) {
        const u32 half = 1u << (r - 1 - s), quarter = half >> 1;
        for (u32 q4 = tid; q4 < (NBF >> 1); q4 += NT) {
            u32 c, pi;
            if (LAST) { pi = q4 & ((R >> 2) - 1); c = q4 >> (r - 2); } else { c = q4 & (CW - 1); pi = q4 >> cwl; }
            const u32 j = pi & (quarter - 1), grp = pi >> (r - 2 - s);
            const u32 u = (grp << (r - s)) + j;
            const u32 i0 = sidx(u, c), i1 = sidx(u + quarter, c), i2 = sidx(u + half, c), i3 = sidx(u + half + quarter, c);
            Fr x0 = sm.ld(i0), x1 = sm.ld(i1), x2 = sm.ld(i2), x3 = sm.ld(i3);
            // stage s: (x0, x2) twiddle index j, (x1, x3) twiddle index j + quarter
            Fr d02 = x0 - x2, d13 = (x1 - x3) * Fr::load_nc(a.wtab + ((size_t)(j + quarter) << s));
            if (j) d02 = d02 * Fr::load_nc(a.wtab + ((size_t)j << s));
            Fr s02 = x0 + x2, s13 = x1 + x3;
            // stage s+1: (s02, s13) and (d02, d13), both with twiddle index j
            Fr e = s02 - s13, f = d02 - d13;
            if (j) {
                const Fr w2 = Fr::load_nc(a.wtab + ((size_t)j << (s + 1)));
                e = e * w2;
                f = f * w2;
            }
            sm.st(i0, s02 + s13);
            sm.st(i1, e);
            sm.st(i2, d02 + d13);
            sm.st(i3, f);
        }
        __syncthreads();
    }
    for (; s < r; s++) {
        const u32 half = 1u << (r - 1 - s);
        for (u32 q = tid; q < NBF; q += NT) {
            u32 c, pi;
            if (LAST) { pi = q & ((R >> 1) - 1); c = q >> (r - 1); } else { c = q & (CW - 1); pi = q >> cwl; }
            u32 j = pi & (half - 1), grp = pi >> (r - 1 - s);
            u32 u = (grp << (r - s)) + j;
            u32 iu = sidx(u, c), iv = sidx(u + half, c);
            Fr x = sm.ld(iu), y = sm.ld(iv);
            Fr d = x - y;
            if (j) d = d * Fr::load_nc(a.wtab + ((size_t)j << s));
            sm.st(iu, x + y);
            sm.st(iv, d);
        }
        __syncthreads();
    }

    // ---- store: row i of the column is at bit-reversed shared position
    for (u32 e = tid; e < TILE; e += NT) {
        u32 c = e & (CW - 1), row = e >> cwl;
        u32 col = col0 + c;
        u32 rrow = __brev(row) >> (32 - r);
        if (r == 0) rrow = 0;
        Fr v = sm.ld(sidx(rrow, c));
        if (LAST) {
            u32 i1 = col & ((1u << a.logN1) - 1), rest = col >> a.logN1;
            size_t nat = (size_t)i1 + (((size_t)rest + ((size_t)row << a.logBrest)) << a.logN1);
            if (a.n_inv) v = v * Fr::load_nc(a.n_inv);
            if (a.coset == 2) {
                u32 m = (u32)(nat % 3);
                if (m) v = v * fr_zeta(3 - (int)m);  // zeta^-m = zeta^(3-m)
            }
            v.store(a.out + nat);
        } else {
            const size_t g = gaddr(row, col);
            v = v * Fr::load_nc(a.tw_full + g);
            v.store(a.out + g);
        }
    }
}

static NttPlan* get_plan(h2b_ctx* ctx, uint32_t log_n, const uint64_t omega[4], int scaled) {
    std::array<uint64_t, 5> key = {omega[0], omega[1], omega[2], omega[3], (uint64_t)log_n | ((uint64_t)(scaled ? 1 : 0) << 32)};
    auto it = ctx->ntt_plans.find(key);
    if (it != ctx->ntt_plans.end()) return it->second;
    const bool domain_root = log_n <= 28 && (memcmp(omega, FR_OMEGA[log_n], 32) == 0 || memcmp(omega, FR_OMEGA_INV[log_n], 32) == 0);
    if (!domain_root) {  // evict the oldest plan of an arbitrary root once the bound is reached
        size_t adhoc = 0;
        auto oldest = ctx->ntt_plans.end();
        for (auto jt = ctx->ntt_plans.begin(); jt != ctx->ntt_plans.end(); ++jt) {
            if (jt->second->domain_root) continue;
            adhoc++;
            if (oldest == ctx->ntt_plans.end() || jt->second->seq < oldest->second->seq) oldest = jt;
        }
        if (adhoc >= NTT_MAX_ADHOC_PLANS) {
            H2B_CUDA(cudaDeviceSynchronize());  // a transform that uses the plan may still be in flight
            if (oldest->second->block) cudaFree(oldest->second->block);
            if (oldest->second->block2) cudaFree(oldest->second->block2);
            delete oldest->second;
            ctx->ntt_plans.erase(oldest);
        }
    }
    static uint64_t plan_seq = 0;
    NttPlan* p = new NttPlan();
    p->domain_root = domain_root;
    p->seq = ++plan_seq;
    struct Guard {  // a failed allocation / launch must not leak the half-built plan
        NttPlan* p;
        ~Guard() {
            if (!p) return;
            if (p->block) cudaFree(p->block);
            if (p->block2) cudaFree(p->block2);
            delete p;
        }
    } guard{p};
    p->log_n = log_n;
    p->npass = log_n <= NTT_MAX_R ? 1 : (log_n <= 2 * NTT_MAX_R ? 2 : 3);
    {
        int rem = (int)log_n;
        for (int t = 0; t < p->npass; t++) {
            int left = p->npass - t;
            p->r[t] = (rem + left - 1) / left;  // larger digits first
            rem -= p->r[t];
        }
        // the last pass reads/writes the longest contiguous rows: give it the largest digit
        if (p->npass > 1) { int tmp = p->r[0]; p->r[0] = p->r[p->npass - 1]; p->r[p->npass - 1] = tmp; }
    }
    p->h = (int)(log_n + 1) / 2;
    size_t n_lo = (size_t)1 << p->h, n_hi = (size_t)1 << (log_n - p->h);
    size_t total = n_lo + n_hi + 1;
    for (int t = 0; t < p->npass; t++) total += (size_t)1 << (p->r[t] > 0 ? p->r[t] - 1 : 0);
    H2B_CUDA(cudaMalloc(&p->block, total * sizeof(Fr)));
    Fr* cur = (Fr*)p->block;
    p->tw_lo = cur; cur += n_lo;
    p->tw_hi = cur; cur += n_hi;
    p->n_inv = cur; cur += 1;
    Fr w;
    memcpy(&w, omega, sizeof(Fr));
    H2B_LAUNCH(ctx, k_pow_table, ceil_div(n_lo, 128), 128, 0, w, (uint64_t)1, (u32)n_lo, p->tw_lo);
    H2B_LAUNCH(ctx, k_pow_table, ceil_div(n_hi, 128), 128, 0, w, (uint64_t)1 << p->h, (u32)n_hi, p->tw_hi);
    H2B_LAUNCH(ctx, k_n_inv, 1, 1, 0, log_n, p->n_inv);
    for (int t = 0; t < p->npass; t++) {
        size_t cnt = (size_t)1 << (p->r[t] > 0 ? p->r[t] - 1 : 0);
        p->wtab[t] = cur; cur += cnt;
        H2B_LAUNCH(ctx, k_pow_table, ceil_div(cnt, 128), 128, 0, w, (uint64_t)1 << (log_n - p->r[t]), (u32)cnt, p->wtab[t]);
    }
    p->scaled = scaled ? 1 : 0;
    if (p->npass > 1) {
        const size_t n = (size_t)1 << log_n;
        H2B_CUDA(cudaMalloc(&p->block2, (size_t)(p->npass - 1) * n * sizeof(Fr)));
        int consumed = 0;
        for (int t = 0; t < p->npass - 1; t++) {
            p->tw_full[t] = (Fr*)p->block2 + (size_t)t * n;
            const int logM = (int)log_n - consumed - p->r[t];
            H2B_LAUNCH(ctx, k_tw_full, ceil_div(n, 256), 256, 0, p->tw_lo, p->tw_hi, p->h, (int)log_n, p->r[t], logM, consumed,
                       (t == 0 && scaled) ? p->n_inv : (const Fr*)nullptr, p->tw_full[t]);
            consumed += p->r[t];
        }
    }
    // the tables are built on whichever stream is current; a later use from another stream (h2b_ctx_set_stream, the side
    // queue) must not overtake the build
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->ntt_plans[key] = p;
    guard.p = nullptr;
    return p;
}

void ntt_free_plans(h2b_ctx* ctx) {
    for (auto& kv : ctx->ntt_plans) {
        if (kv.second->block) cudaFree(kv.second->block);
        if (kv.second->block2) cudaFree(kv.second->block2);
        delete kv.second;
    }
    ctx->ntt_plans.clear();
}

void domain_power_tables(h2b_ctx* ctx, uint32_t k, const void** lo, const void** hi, int* h) {
    H2B_REQUIRE(k >= 1 && k <= 28, "domain_power_tables: k out of range");
    const NttPlan* p = get_plan(ctx, k, FR_OMEGA[k], 0);
    *lo = p->tw_lo;
    *hi = p->tw_hi;
    *h = p->h;
}

void domain_omega(uint32_t k, uint64_t out[4], bool inverse) {
    memcpy(out, inverse ? FR_OMEGA_INV[k] : FR_OMEGA[k], 32);
}

// dst (2^log_n elements, natural order) = NTT_omega(src zero-padded from n_src); src may alias dst.
void ntt_run(h2b_ctx* ctx, const void* d_src, size_t n_src, void* d_dst, uint32_t log_n, const uint64_t omega[4],
             int inverse_scale, int coset_mode) {
    H2B_REQUIRE(log_n <= 28, "ntt: log_n exceeds the two-adicity of Fr (28)");
    const size_t n = (size_t)1 << log_n;
    H2B_REQUIRE(n_src <= n, "ntt: more input elements than the domain size");
    NttPlan* p = get_plan(ctx, log_n, omega, inverse_scale);
    if (!ctx->ntt_attr_set) {  // per context: the attribute belongs to the device the context is bound to
        // up to the whole 227 KB: a transform that runs in the background asks for more shared memory than it uses so that
        // only 1 or 2 of its CTAs fit on an SM (option "ntt.max_ctas_per_sm")
        H2B_CUDA(cudaFuncSetAttribute(k_ntt_pass<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, NTT_SMEM_MAX));
        H2B_CUDA(cudaFuncSetAttribute(k_ntt_pass<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, NTT_SMEM_MAX));
        ctx->ntt_attr_set = true;
    }
    Fr* scratch = nullptr;
    if (p->npass > 1) scratch = (Fr*)ctx->get(WS_NTT_B, n * sizeof(Fr));
    // Tile size: 2^11 elements for large transforms; smaller domains take smaller tiles so that the grid still covers the
    // GPU several times over (2^19: 512 CTAs of 2^10 instead of 256 of 2^11; 2^16: 256 CTAs instead of 32) — the passes are
    // latency-bound there, more resident warps hide the multiplier's dependent chains.
    int r_max = 0;
    for (int t = 0; t < p->npass; t++) r_max = std::max(r_max, p->r[t]);
    const int tile_log = std::min(NTT_TILE_LOG, std::max(r_max, (int)log_n - 10));
    int consumed = 0;
    for (int t = 0; t < p->npass; t++) {
        const bool last = (t == p->npass - 1), first = (t == 0);
        PassArgs a{};
        a.in = first ? (const Fr*)d_src : scratch;
        a.out = last ? (Fr*)d_dst : scratch;
        a.n_in = first ? (u32)n_src : (u32)n;
        a.log_n = (int)log_n;
        a.r = p->r[t];
        a.logM = (int)log_n - consumed - a.r;
        int cols_log = (int)log_n - a.r;
        a.cw_log = tile_log - a.r;
        if (a.cw_log > cols_log) a.cw_log = cols_log;
        if (a.cw_log < 0) a.cw_log = 0;
        a.first = first;
        a.last = last;
        a.logN1 = p->npass > 1 ? p->r[0] : 0;
        a.logBrest = cols_log - a.logN1;
        a.wtab = p->wtab[t];
        a.n_inv = (last && inverse_scale && p->npass == 1) ? p->n_inv : nullptr;  // multi-pass: folded into tw_full[0]
        a.tw_full = last ? nullptr : p->tw_full[t];
        a.coset = coset_mode;
        const unsigned grid = 1u << (cols_log - a.cw_log);
        size_t smem = sizeof(Fr) << (a.r + a.cw_log);
        // background mode: at most opt_ntt_ctas CTAs of this transform per SM, so that the few-CTA kernels of a latency-bound
        // MSM pipeline running beside it always find a free slot (the transform is slower, but hidden)
        if (ctx->opt_ntt_ctas >= 1 && ctx->opt_ntt_ctas <= 2) smem = std::max(smem, (size_t)(NTT_SMEM_MAX / ctx->opt_ntt_ctas - 1024) & ~(size_t)1023);
        const unsigned threads = (unsigned)std::min(NTT_THREADS, std::max(32, (1 << (a.r + a.cw_log)) / 4));
        if (last) H2B_LAUNCH(ctx, k_ntt_pass<true>, grid, threads, smem, a);
        else H2B_LAUNCH(ctx, k_ntt_pass<false>, grid, threads, smem, a);
        consumed += a.r;
    }
}

}  // namespace h2b
