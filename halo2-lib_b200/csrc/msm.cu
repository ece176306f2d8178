// msm.cu — multi-scalar multiplication over BN254 G1 for sm_90a.
//
// Replaces halo2curves-axiom 0.7.3 `msm::best_multiexp(coeffs, bases)` as reached from
// ParamsKZG::commit / commit_lagrange inside create_proof (sole halo2-lib call site of create_proof:
// halo2-base/src/utils/testing.rs:40-48; SURVEY.md §3.3, §8 a2/a4).  The result is the same group element.
//
// Pipeline (no host synchronisation; up to 16 MSMs of one size — the columns a prover phase commits — share ONE pipeline,
// their bucket sets side by side, msm_run_group; the bucket reduction of a lane's group runs on a high-priority stream):
//   k_sort_count      scalars (Montgomery) -> canonical -> signed base-2^c digits -> bucket keys (stored) and a shared
//                     histogram of coarse bins (key >> F) -> one global add per (tile, bin); the last CTA scans the bin
//                     counts and splits every bin into chunks for the fine passes
//   k_sort_partition  writes (low F key bits, table index | table bit | sign) into the bins' regions, one global atomic
//                     per (tile, bin) reserves a tile's run
//   k_sort_fine<0>    per chunk of a bin: shared histogram of its 2^F buckets -> one global add per (chunk, bucket)
//   k_scan_tiles/apply exclusive scan: first sorted position of every bucket
//   k_sort_fine<1>    per chunk: reserves a run per (chunk, bucket), ranks in shared memory, writes the sorted entries
//   k_accumulate      every thread owns EXACTLY L consecutive sorted entries (perfect balance under any
//                     scalar distribution, witness columns are dominated by 0/1/88-bit limbs), gathers the
//                     64-byte affine points with 128-bit loads, XYZZ mixed adds; buckets that end inside
//                     the chunk are written directly, runs cut by a chunk border go to a partial array
//   k_collect         per bucket: add the partials of the chunks it spans; buckets spanning > 64 chunks are
//   k_collect_big1/2  cut into segments summed by whole CTAs
//   k_rowcol_sums     bucket grid 2^mh x 2^ml: one CTA of 32 lane-quads per row sum / column sum (quad.cuh)
//   k_rowcol_weights  lo * R_lo and (2^ml hi + 1) * C_hi by 4-lane double-and-add, one quad per point
//   k_weighted_final  the two sums of the weighted points; the last CTA of every MSM adds them (Horner over bucket
//                     sets for ad-hoc bases) and stores that MSM's Jacobian result
//
// Fixed bases (the SRS): `table[w*n + i] = 2^(c*w) * P_i` is built once per SRS (k_precompute_level), so all
// windows of a scalar fall into ONE bucket set: no per-window reduction and no final doublings.
#include "curve.cuh"
#include "quad.cuh"
#include "h2b_internal.cuh"

namespace h2b {

static constexpr u32 SIGN_BIT = 0x80000000u;
static constexpr int ACC_L_DEFAULT = 32;  // upper bound of the sorted entries per accumulate thread (see k_accumulate)
static constexpr int BIG_PARTIALS = 64;  // buckets spanning more chunks than this are summed by a whole CTA
// A *group* of MSMs over the same domain size runs through ONE pipeline: the bucket sets of the g-th MSM follow those of
// the (g-1)-th in one bucket array, so the sort, the accumulation and the latency-bound bucket reduction are launched once
// per group (a prover phase commits 1..13 columns at once) instead of once per column.
static constexpr int MSM_MAX_GROUP = 16;
struct MsmScalars { const uint64_t* p[MSM_MAX_GROUP]; };
// The MSMs of a group read at most TWO distinct tables (the SRS has two bases); bit 30 of a sorted entry selects one.
static constexpr u32 TABLE_BIT = 0x40000000u;

// ------------------------------------------------------------------------------------------------ digits + bucket sort
// Signed base-2^c recoding of one canonical scalar; calls f(w, digit_magnitude (0..2^(c-1)), negative) for every
// window, zero digits included.  W*c >= 255 so the last carry is absorbed.
template <class F>
__device__ __forceinline__ void for_each_digit(const Fr& s, int c, int W, F&& f) {
    const u32 half = 1u << (c - 1);
    const u32 mask = (1u << c) - 1u;
    u32 carry = 0;
    for (int w = 0; w < W; w++) {
        int bit = w * c;
        u32 raw = 0;
        if (bit < 256) {
            int limb = bit >> 5, off = bit & 31;
            u32 lo = 0, hi = 0;  // dynamic limb index on a register array: select through a small unrolled scan
#pragma unroll
            for (int t = 0; t < 8; t++) {
                if (t == limb) lo = s.l[t];
                if (t == limb + 1) hi = s.l[t];
            }
            u64 v = ((u64)hi << 32) | lo;
            raw = (u32)(v >> off) & mask;
        }
        u32 d = raw + carry;
        bool neg = false;
        if (d > half) {
            d = (1u << c) - d;
            neg = true;
            carry = 1;
        } else {
            carry = 0;
        }
        f(w, d, neg);
    }
}

// Counter increment with two fast paths for hot counters.  (1) all active lanes of the warp hit the SAME counter
// (constant columns, padding runs): one atomic per warp.  (2) lanes whose digit is tiny (|d| <= 4: bit-valued and
// small-constant witness cells, the hot buckets of real advice columns) or in the top window (its digit only spans the
// few leading bits of the scalar) are grouped by __match_any_sync and issue
// one atomic per distinct counter.  Everything else uses a plain atomic; uniform digits are almost never tiny, so
// the common case pays nothing for (2).  All 32 lanes must call; returns the slot of the lane.
__device__ __forceinline__ u32 warp_agg_add(u32* counters, u32 key, bool active, bool tiny) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned mask = __ballot_sync(0xffffffffu, active);
    if (!active) return 0;
    const u32 kmin = __reduce_min_sync(mask, key), kmax = __reduce_max_sync(mask, key);
    if (kmin == kmax) {
        const int leader = __ffs(mask) - 1;
        u32 base = 0;
        if ((int)lane == leader) base = atomicAdd(counters + key, (u32)__popc(mask));
        base = __shfl_sync(mask, base, leader);
        return base + __popc(mask & ((1u << lane) - 1));
    }
    const unsigned tmask = __ballot_sync(mask, tiny);
    if (tiny) {
        const unsigned peers = __match_any_sync(tmask, key);
        const int leader = __ffs(peers) - 1;
        u32 base = 0;
        if ((int)lane == leader) base = atomicAdd(counters + key, (u32)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        return base + __popc(peers & ((1u << lane) - 1));
    }
    return atomicAdd(counters + key, 1u);
}

// Two-level sort of the non-zero digits by bucket key.  A one-level counting sort pays a global atomic and a scattered 4-byte
// store per digit (7.9 M of each per 2^19 MSM).  Here the per-digit counting and ranking happen in shared memory, a global
// atomic stands for a whole (tile, bin) or (chunk, bucket) run, and every pass stages its entries in shared memory sorted by
// destination so that the stores go out in contiguous runs.
//   coarse bins  bin = key >> F, nbins <= SORT_BINS_MAX (F chosen per shape by msm_run_group); fine: the 2^F keys of a bin
//   k_sort_count      per tile of scalars: recodes, stores every digit's key (coalesced, [msm][window][scalar]) and
//                     counts the bins in shared memory -> bin_count (one global add per non-empty bin).  The only kernel
//                     that reads the scalars.  Its last CTA scans bin_count into bin_base and cuts every bin into chunks
//                     for the fine passes.
//   k_sort_partition  per tile of keys: reserves a run per (tile, bin) and writes (key & (2^F - 1), entry) pairs into the
//                     bins' regions of tmp_low / tmp_val
//   k_sort_fine<0>    per chunk of one bin: shared histogram of the bin's 2^F buckets -> hist (one add per bucket)
//   k_scan_tiles/apply exclusive scan of hist: off[] (first sorted position of every bucket), cursor[], off[nb], L
//   k_sort_fine<1>    per chunk: reserves a run per (chunk, bucket) from cursor[] and writes the chunk's entries there
// Entry order inside a bucket depends on the order of the atomics (as in any counting sort on the GPU); the sum does not.
static constexpr int SORT_BINS_MAX = 4096;  // coarse bins at most (2^23 buckets with F = 11)
static constexpr int SORT_F_MAX = 11;       // fine buckets per bin at most 2^11: a chunk still averages 4 entries per bucket
static constexpr int SORT_PART_TS = 256;    // scalars per CTA of k_sort_partition
static constexpr u32 SORT_CHUNK = 8192;     // entries per CTA of the fine passes
static constexpr int SORT_FINE_U = 4;       // entries per thread and step of the fine passes (loads in flight)
static constexpr int SORT_PART_SMEM_MAX = 2 * SORT_BINS_MAX * 4 + 43 * SORT_PART_TS * 12;  // W <= 43 (ad-hoc c = 6)
static constexpr int SORT_FINE_SMEM = (2 << SORT_F_MAX) * 4 + SORT_CHUNK * 6;

// Exclusive scan of a[0, len) in shared memory by the whole block (blockDim.x a multiple of 32).  `a` must be complete
// (a __syncthreads() before the call); returns the total after a final __syncthreads().
__device__ u32 block_exclusive_scan(u32* a, u32 len, u32* wsum /* [32] */) {
    const u32 t = threadIdx.x, nt = blockDim.x, per = (len + nt - 1) / nt;
    const u32 b0 = min(t * per, len), b1 = min(b0 + per, len);
    u32 sum = 0;
    for (u32 j = b0; j < b1; j++) sum += a[j];
    u32 inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
        if ((t & 31) >= (u32)d) inc += o;
    }
    if ((t & 31) == 31) wsum[t >> 5] = inc;
    __syncthreads();
    u32 run = inc - sum, total = 0;
    for (u32 w = 0; w < nt / 32; w++) {
        if (w < (t >> 5)) run += wsum[w];
        total += wsum[w];
    }
    for (u32 j = b0; j < b1; j++) {
        const u32 v = a[j];
        a[j] = run;
        run += v;
    }
    __syncthreads();
    return total;
}

// Window w belongs to bucket set w / q and table level w % q.  Zero digits are dropped.  blockIdx.y = MSM of the group; its
// bucket sets start at bucket blockIdx.y * spm * nbw (spm = sets per MSM).  q is W (tabulated bases) or 1 (ad-hoc bases):
// both are answered without an integer division.
__device__ __forceinline__ u32 window_set(int w, int q) { return q == 1 ? (u32)w : (w < q ? 0u : (u32)(w / q)); }
__device__ __forceinline__ u32 window_level(int w, int q) { return q == 1 ? 0u : (w < q ? (u32)w : (u32)(w % q)); }
__device__ __forceinline__ u32 digit_key(u32 msm, int w, int q, u32 nbw, u32 spm, u32 d) {
    return msm * spm * nbw + window_set(w, q) * nbw + (d - 1);
}
static constexpr u32 NO_DIGIT = ~0u;  // k_sort_count's key of a zero digit

// One scalar per thread.  The last CTA to finish turns the bin counts into bin_base[b] = first position of bin b
// (bin_base[nbins] = entry count), bin_cursor = bin_base (consumed by k_sort_partition) and chunk_pre[b] = first fine-pass
// chunk of bin b (chunk_pre[nbins] = chunk count).  `done` is zero at the launch.
__global__ void __launch_bounds__(256) k_sort_count(const __grid_constant__ MsmScalars cols, u32 n, int c, int W, int q, u32 nbw,
                                                    u32 spm, int F, u32 nbins, u32* __restrict__ bin_count,
                                                    u32* __restrict__ keys, u32* __restrict__ done, u32* __restrict__ bin_base,
                                                    u32* __restrict__ bin_cursor, u32* __restrict__ chunk_pre) {
    __shared__ u32 h[SORT_BINS_MAX], nch[SORT_BINS_MAX];
    __shared__ u32 wsum[32];
    __shared__ bool is_last;
    for (u32 b = threadIdx.x; b < nbins; b += blockDim.x) h[b] = 0;
    __syncthreads();
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    Fr s = Fr::zero();
    if (live) s = Fr::load_nc(cols.p[blockIdx.y] + 4 * (size_t)i).from_mont();  // canonical integer, as `to_repr()` gives
    for_each_digit(s, c, W, [&](int w, u32 d, bool neg) {
        const bool active = live && d != 0;
        const u32 key = active ? digit_key(blockIdx.y, w, q, nbw, spm, d) : 0;
        // tiny digits and the (narrow) top window are where hot buckets come from: group them before the atomic
        warp_agg_add(h, key >> F, active, d <= 4 || w == W - 1);
        if (live) keys[((size_t)blockIdx.y * W + w) * n + i] = active ? key | (neg ? SIGN_BIT : 0u) : NO_DIGIT;
    });
    __syncthreads();
    for (u32 b = threadIdx.x; b < nbins; b += blockDim.x)
        if (h[b]) atomicAdd(bin_count + b, h[b]);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(done, 1u) == gridDim.x * gridDim.y - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (u32 b = threadIdx.x; b < nbins; b += blockDim.x) {
        h[b] = __ldcg(bin_count + b);
        nch[b] = (h[b] + SORT_CHUNK - 1) / SORT_CHUNK;
    }
    __syncthreads();
    const u32 total = block_exclusive_scan(h, nbins, wsum);
    const u32 chunks = block_exclusive_scan(nch, nbins, wsum);
    for (u32 b = threadIdx.x; b < nbins; b += blockDim.x) {
        bin_base[b] = h[b];
        bin_cursor[b] = h[b];
        chunk_pre[b] = nch[b];
    }
    if (threadIdx.x == 0) {
        bin_base[nbins] = total;
        chunk_pre[nbins] = chunks;
    }
}

// Tile = SORT_PART_TS scalars, one per thread.  The keys k_sort_count recorded wait in shared memory (with their rank inside
// the tile's run of the bin) until one global atomic per non-empty bin has reserved the tile's runs; then they are put in bin
// order in shared memory and stored in contiguous runs.
__global__ void __launch_bounds__(SORT_PART_TS) k_sort_partition(const u32* __restrict__ keys, u32 n, int W, int q, u32 nbw,
                                                                 u32 table_mask, int F, u32 nbins, u32* __restrict__ bin_cursor,
                                                                 uint16_t* __restrict__ tmp_low, u32* __restrict__ tmp_val) {
    extern __shared__ u32 sdyn[];
    __shared__ u32 wsum[32];
    const u32 ts = SORT_PART_TS, t = threadIdx.x, ne = (u32)W * ts;
    u32* h = sdyn;                                 // [nbins] count, then first position of the bin in the tile's order
    u32* dlt = h + nbins;                          // [nbins] global position - tile position
    u32* skey = dlt + nbins;                       // [W][ts] key | sign, NO_DIGIT for a zero digit
    u32* okey = skey + ne;                         // [ne] key | sign in bin order
    uint16_t* srank = (uint16_t*)(okey + ne);      // [W][ts] rank inside the tile's run of the bin
    uint16_t* osrc = srank + ne;                   // [ne] w << 8 | thread, in bin order
    for (u32 b = t; b < nbins; b += ts) h[b] = 0;
    __syncthreads();
    const u32 i = blockIdx.x * ts + t;
    const bool live = i < n;
    const u32* __restrict__ mk = keys + (size_t)blockIdx.y * W * n + i;
#pragma unroll 4
    for (int w = 0; w < W; w++) skey[w * ts + t] = live ? mk[(size_t)w * n] : NO_DIGIT;  // independent loads first
    for (int w = 0; w < W; w++) {
        const u32 k = skey[w * ts + t], key = k & ~SIGN_BIT;
        // digit - 1 is the key's offset in its bucket set: the same grouping of hot buckets as in k_sort_count
        const u32 r = warp_agg_add(h, key >> F, k != NO_DIGIT, (key & (nbw - 1)) < 4 || w == W - 1);
        srank[w * ts + t] = (uint16_t)r;
    }
    __syncthreads();
    for (u32 b = t; b < nbins; b += ts) dlt[b] = h[b] ? atomicAdd(bin_cursor + b, h[b]) : 0u;
    const u32 total = block_exclusive_scan(h, nbins, wsum);
    for (u32 b = t; b < nbins; b += ts) dlt[b] -= h[b];
    for (int w = 0; w < W; w++) {
        const u32 k = skey[w * ts + t];
        if (k == NO_DIGIT) continue;
        const u32 p = h[(k & ~SIGN_BIT) >> F] + srank[w * ts + t];
        okey[p] = k;
        osrc[p] = (uint16_t)((w << 8) | t);
    }
    __syncthreads();
    const u32 tbit = ((table_mask >> blockIdx.y) & 1u) ? TABLE_BIT : 0u;
    const u32 fmask = (1u << F) - 1u;
    for (u32 j = t; j < total; j += ts) {
        const u32 k = okey[j], key = k & ~SIGN_BIT, src = osrc[j];
        const u32 pos = dlt[key >> F] + j;
        tmp_low[pos] = (uint16_t)(key & fmask);
        tmp_val[pos] = (window_level(src >> 8, q) * n + blockIdx.x * ts + (src & 255u)) | tbit | (k & SIGN_BIT);
    }
}

// The fine passes run one CTA per chunk of SORT_CHUNK entries of one bin (chunks never straddle bins).  False: no such chunk.
__device__ __forceinline__ bool sort_chunk(const u32* __restrict__ chunk_pre, const u32* __restrict__ bin_base, u32 nbins,
                                           u32& bin, u32& s, u32& e) {
    const u32 g = blockIdx.x;
    if (g >= chunk_pre[nbins]) return false;
    u32 lo = 0, hi = nbins;  // chunk_pre[lo] <= g < chunk_pre[hi]
    while (hi - lo > 1) {
        const u32 mid = (lo + hi) >> 1;
        if (chunk_pre[mid] <= g) lo = mid; else hi = mid;
    }
    bin = lo;
    s = bin_base[lo] + (g - chunk_pre[lo]) * SORT_CHUNK;
    e = min(s + SORT_CHUNK, bin_base[lo + 1]);
    return true;
}

// MODE 0: hist[bin * 2^F + low] += the chunk's count of that bucket.
// MODE 1: reserves the chunk's run of every bucket from cursor[], puts the chunk in bucket order in shared memory and stores
// it to vals in contiguous runs.
template <int MODE>
__global__ void __launch_bounds__(512) k_sort_fine(const u32* __restrict__ chunk_pre, const u32* __restrict__ bin_base, u32 nbins,
                                                   int F, const uint16_t* __restrict__ tmp_low, const u32* __restrict__ tmp_val,
                                                   u32* __restrict__ counters, u32* __restrict__ vals) {
    extern __shared__ u32 h[];  // [2^F] count, then (MODE 1) running position in the chunk's bucket order
    __shared__ u32 wsum[32];
    u32 bin, s, e;
    if (!sort_chunk(chunk_pre, bin_base, nbins, bin, s, e)) return;
    const u32 nf = 1u << F, t = threadIdx.x;
    for (u32 j = t; j < nf; j += blockDim.x) h[j] = 0;
    __syncthreads();
    // all 32 lanes of a warp call warp_agg_add: the loop bound is uniform.  A hot bucket fills whole warps.  SORT_FINE_U
    // independent loads are issued before their atomics.
    const u32 bd = blockDim.x;
    for (u32 i0 = s; i0 < e; i0 += SORT_FINE_U * bd) {
        u32 lw[SORT_FINE_U];
#pragma unroll
        for (int u = 0; u < SORT_FINE_U; u++) lw[u] = i0 + u * bd + t < e ? tmp_low[i0 + u * bd + t] : 0u;
#pragma unroll
        for (int u = 0; u < SORT_FINE_U; u++) warp_agg_add(h, lw[u], i0 + u * bd + t < e, false);
    }
    __syncthreads();
    u32* ctr = counters + ((size_t)bin << F);
    if (MODE == 0) {
        for (u32 j = t; j < nf; j += blockDim.x)
            if (h[j]) atomicAdd(ctr + j, h[j]);
        return;
    }
    u32* dlt = h + nf;                              // [2^F] global position - chunk position
    u32* oval = dlt + nf;                           // [chunk] entries in bucket order
    uint16_t* olow = (uint16_t*)(oval + SORT_CHUNK);  // [chunk] their buckets
    for (u32 j = t; j < nf; j += blockDim.x) dlt[j] = h[j] ? atomicAdd(ctr + j, h[j]) : 0u;
    block_exclusive_scan(h, nf, wsum);
    for (u32 j = t; j < nf; j += blockDim.x) dlt[j] -= h[j];
    __syncthreads();  // h becomes the running position below
    for (u32 i0 = s; i0 < e; i0 += SORT_FINE_U * bd) {
        u32 lw[SORT_FINE_U], vw[SORT_FINE_U];
#pragma unroll
        for (int u = 0; u < SORT_FINE_U; u++) {
            const u32 i = i0 + u * bd + t;
            lw[u] = i < e ? tmp_low[i] : 0u;
            vw[u] = i < e ? tmp_val[i] : 0u;
        }
#pragma unroll
        for (int u = 0; u < SORT_FINE_U; u++) {
            const bool active = i0 + u * bd + t < e;
            const u32 p = warp_agg_add(h, lw[u], active, false);
            if (active) {
                oval[p] = vw[u];
                olow[p] = (uint16_t)lw[u];
            }
        }
    }
    __syncthreads();
    for (u32 j = t; j < e - s; j += blockDim.x) vals[dlt[olow[j]] + j] = oval[j];
}

// Exclusive scan of the histogram in two launches.  Tile = 2048 counters per CTA.
// k_scan_tiles: off[b] = exclusive prefix inside the tile, tile_sums[tile] = tile total.
// k_scan_apply: adds the sum of the preceding tile totals; cursor[b] = off[b]; off[nb] = grand total.
static constexpr int SCAN_TILE = 2048;
__global__ void __launch_bounds__(256) k_scan_tiles(const u32* __restrict__ hist, u32 nb, u32* __restrict__ off,
                                                    u32* __restrict__ tile_sums) {
    __shared__ u32 sh[SCAN_TILE];
    __shared__ u32 wsum[8];
    const u32 base = blockIdx.x * SCAN_TILE, t = threadIdx.x;
    for (u32 e = t; e < SCAN_TILE; e += 256) sh[e] = (base + e < nb) ? hist[base + e] : 0;  // coalesced
    __syncthreads();
    u32 v[8], sum = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { v[j] = sh[t * 8 + j]; sum += v[j]; }
    // block exclusive scan of the 256 per-thread sums: warp shuffle scan + scan of the 8 warp totals
    u32 inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        u32 o = __shfl_up_sync(0xffffffffu, inc, d);
        if ((t & 31) >= (u32)d) inc += o;
    }
    if ((t & 31) == 31) wsum[t >> 5] = inc;
    __syncthreads();
    u32 wbase = 0;
    for (u32 w = 0; w < (t >> 5); w++) wbase += wsum[w];
    u32 run = wbase + inc - sum;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; j++) { sh[t * 8 + j] = run; run += v[j]; }
    __syncthreads();
    for (u32 e = t; e < SCAN_TILE; e += 256)
        if (base + e < nb) off[base + e] = sh[e];
    if (t == 255) tile_sums[blockIdx.x] = run;
}
__global__ void __launch_bounds__(256) k_scan_apply(u32 nb, u32 ntiles, const u32* __restrict__ tile_sums,
                                                    u32* __restrict__ off, u32* __restrict__ cursor, u32 slots,
                                                    u32 l_min, u32 l_max, u32* __restrict__ d_L) {
    __shared__ u32 red[256];
    const u32 t = threadIdx.x;
    u32 s = 0;
    for (u32 j = t; j < blockIdx.x; j += 256) s += tile_sums[j];  // sum of the preceding tiles
    red[t] = s;
    __syncthreads();
    for (int d = 128; d >= 1; d >>= 1) {
        if (t < (u32)d) red[t] += red[t + d];
        __syncthreads();
    }
    const u32 add = red[0], base = blockIdx.x * SCAN_TILE;
    for (u32 e = t; e < SCAN_TILE; e += 256)
        if (base + e < nb) {
            u32 o = off[base + e] + add;
            off[base + e] = o;
            cursor[base + e] = o;
        }
    if (blockIdx.x == ntiles - 1 && t == 0) {
        const u32 mv = add + tile_sums[ntiles - 1];
        off[nb] = mv;
        // chunk length for k_accumulate: whole waves of equally long chunks (see k_accumulate)
        u32 L = l_max;
        if (mv < l_max * slots) {  // less than one full wave of l_max-chunks: spread the entries over every slot
            L = (mv + slots - 1) / slots;
            if (L < l_min) L = l_min;
        }
        *d_L = L;
    }
}

// ------------------------------------------------------------------------------------------------ accumulate
__device__ __forceinline__ Affine load_signed(const Affine* __restrict__ table, const Affine* __restrict__ table_b, u32 val) {
    Affine p = Affine::load(((val & TABLE_BIT) ? table_b : table) + (val & ~(SIGN_BIT | TABLE_BIT)));
    if (val & SIGN_BIT) p.y = p.y.neg();
    return p;
}

__device__ __forceinline__ u32 offs(const u32* __restrict__ off, u32 b) { return __ldg(off + b); }
// first bucket b in [lo, nb) with off[b + 1] > pos  (the bucket that owns sorted position pos)
__device__ __forceinline__ u32 bucket_of(const u32* __restrict__ off, u32 lo, u32 nb, u32 pos) {
    u32 hi = nb;
    while (lo < hi) {
        u32 mid = (lo + hi) >> 1;
        if (offs(off, mid + 1) > pos) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// Chunk length L is chosen ON THE DEVICE by k_scan_apply once the number of entries is known (zero digits are
// dropped, so it depends on the scalars): 32 normally; when the entries would not even fill one wave of
// 32-entry chunks (sparse witness columns, small shards) L = ceil(entries / slots), slots = resident threads of
// this kernel, so that every SM is busy.  (Whole-wave balancing of dense columns was measured: no gain, the
// kernel is multiplier-bound and a partially filled last wave simply runs faster.)
// Entry i is the table point vals[i] (index | table bit | sign).
__global__ void __launch_bounds__(128, 4) k_accumulate(const u32* __restrict__ vals, const u32* __restrict__ off,
                                                       u32 nb_total, const u32* __restrict__ d_L,
                                                       const Affine* __restrict__ table, const Affine* __restrict__ table_b,
                                                       XYZZ* __restrict__ buckets, XYZZ* __restrict__ partials) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 L = __ldg(d_L);
    const u32 mv = offs(off, nb_total);  // number of entries (non-zero digits)
    const u64 cs64 = (u64)t * L;
    if (cs64 >= mv) return;
    const u32 cs = (u32)cs64;
    const u32 ce = (mv - cs < (u32)L) ? mv : cs + L;
    u32 cur = bucket_of(off, 0, nb_total, cs);
    u32 run_end = offs(off, cur + 1);
    auto fetch = [&](u32 i) -> Affine { return load_signed(table, table_b, __ldg(vals + i)); };
    XYZZ acc = XYZZ::identity();
    Affine p = fetch(cs);
    for (u32 i = cs; i < ce; i++) {
        Affine pn;
        const bool more = (i + 1 < ce);
        if (more) pn = fetch(i + 1);  // prefetch the next point while this add runs
        xyzz_madd(acc, p);
        if (!more || i + 1 == run_end) {
            // the run of bucket `cur` ends here (inside this chunk or at its border)
            const u32 s = offs(off, cur);
            if (s >= cs && run_end - cs <= (u32)L) acc.store(buckets + cur);    // bucket lies inside the chunk
            else if (s <= cs) acc.store(partials + 2 * (size_t)t);              // covers the chunk start
            else acc.store(partials + 2 * (size_t)t + 1);                        // starts inside, runs past the end
            acc = XYZZ::identity();
            if (more) {  // next non-empty bucket: a few linear steps, then binary search (long empty gaps)
                u32 b = cur + 1;
                int steps = 0;
                while (offs(off, b + 1) <= i + 1) {
                    b++;
                    if (++steps == 4) { b = bucket_of(off, b, nb_total, i + 1); break; }
                }
                cur = b;
                run_end = offs(off, cur + 1);
            }
        }
        if (more) p = pn;
    }
}

__device__ __forceinline__ const XYZZ* partial_of(const XYZZ* partials, u32 s, u32 t, u32 L) {
    return (s <= t * L) ? partials + 2 * (size_t)t : partials + 2 * (size_t)t + 1;
}

// one thread per bucket: empty -> identity; spans several chunks -> add their partials
__global__ void __launch_bounds__(128) k_collect(const u32* __restrict__ off, u32 nb_total, const u32* __restrict__ d_L,
                                                 const XYZZ* __restrict__ partials, XYZZ* __restrict__ buckets,
                                                 u32* __restrict__ big_list, u32* __restrict__ big_count) {
    u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb_total) return;
    const u32 L = __ldg(d_L);
    const u32 s = offs(off, b), e = offs(off, b + 1);
    if (s == e) {
        XYZZ::identity().store(buckets + b);
        return;
    }
    const u32 t_lo = s / L, t_hi = (e - 1) / L;
    if (t_lo == t_hi) return;  // written by k_accumulate
    if (t_hi - t_lo + 1 > (u32)BIG_PARTIALS) {
        big_list[atomicAdd(big_count, 1u)] = b;
        return;
    }
    XYZZ acc = XYZZ::load(partial_of(partials, s, t_lo, L));
    for (u32 t = t_lo + 1; t <= t_hi; t++) xyzz_add(acc, XYZZ::load(partials + 2 * (size_t)t));
    acc.store(buckets + b);
}

// Hot buckets (e.g. digit 1 of a bit-valued witness column: a quarter of all entries) span thousands of chunks.
// Stage 1: the partials of every big bucket are cut into segments of 64; one CTA (64 lane-quads) sums a segment.
// Stage 2: one CTA per big bucket sums its segment sums.  Work lists are walked on the device (counts are only
// known there); `seg` needs one slot per 64 chunk partials overall.
static constexpr int BIG_SEG = 64;
__global__ void __launch_bounds__(256) k_collect_big1(const u32* __restrict__ off, const u32* __restrict__ d_L, const XYZZ* __restrict__ partials,
                                                      const u32* __restrict__ big_list, const u32* __restrict__ big_count,
                                                      XYZZ* __restrict__ seg) {
    __shared__ XYZZ sh[8];
    const u32 nbig = *big_count;
    const u32 L = __ldg(d_L);
    const u32 qid = threadIdx.x >> 2;
    u32 seg_base = 0;  // running number of segments of the buckets before j
    u32 g = blockIdx.x;  // next segment of this CTA (segments are numbered across all big buckets)
    for (u32 j = 0; j < nbig; j++) {
        const u32 b = big_list[j];
        const u32 s = offs(off, b), e = offs(off, b + 1);
        const u32 t_lo = s / L, t_hi = (e - 1) / L;
        const u32 cnt = t_hi - t_lo + 1, nseg = (cnt + BIG_SEG - 1) / BIG_SEG;
        for (; g < seg_base + nseg; g += gridDim.x) {
            const u32 t = t_lo + (g - seg_base) * BIG_SEG + qid;
            XYZZ v = XYZZ::identity();
            if (t <= t_hi) v = XYZZ::load(partial_of(partials, s, t, L));
            v = quad_block_sum(v, sh);
            if (threadIdx.x == 0) v.store(seg + g);
            __syncthreads();
        }
        seg_base += nseg;
    }
}
__global__ void __launch_bounds__(256) k_collect_big2(const u32* __restrict__ off, const u32* __restrict__ d_L, const XYZZ* __restrict__ seg,
                                                      XYZZ* __restrict__ buckets, const u32* __restrict__ big_list,
                                                      const u32* __restrict__ big_count) {
    __shared__ XYZZ sh[8];
    const u32 nbig = *big_count;
    const u32 L = __ldg(d_L);
    const u32 qid = threadIdx.x >> 2;
    u32 seg_base = 0;
    for (u32 j = 0; j < nbig; j++) {
        const u32 b = big_list[j];
        const u32 s = offs(off, b), e = offs(off, b + 1);
        const u32 cnt = (e - 1) / L - s / L + 1, nseg = (cnt + BIG_SEG - 1) / BIG_SEG;
        if (j % gridDim.x == blockIdx.x) {
            XYZZ acc = XYZZ::identity();
            for (u32 g = qid; g < nseg; g += 64) quad_add_nl(acc, XYZZ::load(seg + seg_base + g));
            acc = quad_block_sum(acc, sh);
            if (threadIdx.x == 0) acc.store(buckets + b);
            __syncthreads();
        }
        seg_base += nseg;
    }
}

// ------------------------------------------------------------------------------------------------ bucket reduce
// V = sum_b (b+1) * B_b over one bucket set of 2^m buckets, arranged as a 2^mh x 2^ml grid (b = hi * 2^ml + lo):
//     V = sum_b B_b  +  sum_lo lo * R_lo  +  2^ml * sum_hi hi * C_hi ,   R_lo = sum_hi B[hi][lo],  C_hi = sum_lo B[hi][lo].
// A running sum over 2^16 buckets is a dependency chain of ~10^5 point additions; this form has depth
// ~(2^mh / 32 + 5) for the row/column sums (one warp each, shuffle tree), ~2*ml for the small scalar
// multiplications lo * R_lo / hi * C_hi (one thread each) and ~10 for the block sums and the final doublings.
// One CTA of 128 threads (32 lane-quads, quad.cuh) per row sum R_lo / column sum C_hi: every quad adds its
// stride-32 share of the row (column), then the 32 quads are summed and the result is multiplied by its weight.
// rc[set] = [ lo * R_lo (2^ml) | (2^ml hi + 1) * C_hi (2^mh) | C_hi (2^mh) ] after k_rowcol_weights.
__global__ void __launch_bounds__(128) k_rowcol_sums(const XYZZ* __restrict__ buckets, int ml, int mh, u32 nsets,
                                                     XYZZ* __restrict__ rc) {
    __shared__ XYZZ sh[4];
    const u32 per_set = (1u << ml) + (1u << mh);
    const u32 set = blockIdx.x / per_set, idx = blockIdx.x % per_set;
    const u32 qid = threadIdx.x >> 2;
    const XYZZ* base = buckets + ((size_t)set << (ml + mh));
    XYZZ acc = XYZZ::identity();
    if (idx < (1u << ml)) {  // row sum over hi, stride 2^ml
        for (u32 hi = qid; hi < (1u << mh); hi += 32) quad_add(acc, XYZZ::load(base + ((size_t)hi << ml) + idx));
    } else {  // column sum over lo, contiguous
        const u32 hi = idx - (1u << ml);
        for (u32 lo = qid; lo < (1u << ml); lo += 32) quad_add(acc, XYZZ::load(base + ((size_t)hi << ml) + lo));
    }
    acc = quad_block_sum<true>(acc, sh);
    // quad 0 of warp 0 holds the sum.  The weights (lo for a row, hi for a column) are applied by k_rowcol_weights: a
    // double-and-add chain on ONE quad would keep this CTA's four warps resident for as long again, and with the bucket
    // sets of a whole group of MSMs in one launch the CTAs no longer fit in one wave.
    if (threadIdx.x == 0) {
        const bool is_row = idx < (1u << ml);
        XYZZ* out = rc + (size_t)set * ((1u << ml) + 2 * (1u << mh));
        acc.store(is_row ? out + idx : out + (1u << mh) + idx);  // rows in place; plain column sums in the third section
    }
}
// rc[set] = [ R_lo | . | C_hi ]  ->  [ lo * R_lo | (2^ml hi + 1) * C_hi | C_hi ]: one lane-quad per point, 4-lane double-and-add
__global__ void __launch_bounds__(128) k_rowcol_weights(XYZZ* __restrict__ rc, int ml, int mh, u32 nsets) {
    const u32 per_set = (1u << ml) + (1u << mh);
    const u32 q = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;  // quads never straddle the bound: blockDim.x % 4 == 0
    if (q >= nsets * per_set) return;
    const u32 set = q / per_set, idx = q % per_set;
    const bool is_row = idx < (1u << ml);
    XYZZ* base = rc + (size_t)set * ((1u << ml) + 2 * (1u << mh));
    // a column sum carries its own share of V = sum_b (b + 1) B_b in one weight: 2^ml * hi (its index) + 1 (the plain sum
    // of all buckets), so that the final kernel has nothing left but two sums and one addition
    const u32 weight = is_row ? idx : (((idx - (1u << ml)) << ml) + 1u);
    const XYZZ p = XYZZ::load(is_row ? base + idx : base + (1u << mh) + idx);
    const XYZZ w = quad_small_mul<true>(p, weight, is_row ? ml : ml + mh);
    if ((threadIdx.x & 3) == 0) w.store(base + idx);
}

__device__ __forceinline__ void store_jacobian(const XYZZ& p, void* out) {
    // (X, Y, ZZ, ZZZ) -> Jacobian with Z = ZZ*ZZZ:  X_j = X*ZZ*ZZZ^2, Y_j = Y*ZZ^3*ZZZ^2   (no inversion)
    char* o = reinterpret_cast<char*>(out);
    if (p.is_identity()) {
        Fq::zero().store(o);
        Fq::one().store(o + 32);
        Fq::zero().store(o + 64);
        return;
    }
    Fq z = p.zz * p.zzz;
    Fq a = p.zz * p.zzz.sqr();  // ZZ * ZZZ^2
    (p.x * a).store(o);
    (p.y * a * p.zz.sqr()).store(o + 32);
    z.store(o + 64);
}

// S_lo = sum of rc[0 .. 2^ml) (weighted row sums), S_hi = sum of rc[2^ml .. 2^ml + 2^mh) (column sums weighted with
// 2^ml hi + 1): plain sums of 64 x 4 points per CTA (one lane-quad adds 4 of them).  CTAs of a set: [0, sub_lo) -> S_lo, then
// sub_hi CTAs -> S_hi.  `nsets` = sets of ONE MSM; the grid covers gridDim.x / (nsets * cta_per_set) MSMs (a group, see
// MsmScalars): the last CTA of every MSM to finish adds the CTA partials, forms V_set = S_lo + S_hi, runs Horner over the
// sets (`shift` doublings between consecutive sets; one set when the bases are tabulated) and stores that MSM's Jacobian
// result at out + 96 * msm.
static constexpr int WQ = 256;  // points per CTA of k_weighted_final (64 quads x 4)
__global__ void __launch_bounds__(256) k_weighted_final(const XYZZ* __restrict__ rc, int ml, int mh, u32 nsets, int shift,
                                                        XYZZ* __restrict__ parts, u32* __restrict__ done,
                                                        void* __restrict__ out) {
    __shared__ XYZZ sh[8];
    __shared__ XYZZ comb[2];
    __shared__ XYZZ vsets[64];
    __shared__ u32 is_last;
    const u32 sub_lo = ((1u << ml) + WQ - 1) / WQ, sub_hi = ((1u << mh) + WQ - 1) / WQ;
    const u32 cta_per_set = sub_lo + sub_hi;
    const u32 set = blockIdx.x / cta_per_set, c = blockIdx.x % cta_per_set;  // set counts across the MSMs of the group
    const u32 msm = set / nsets;
    const u32 kind = c < sub_lo ? 0 : 1;
    const u32 sub = kind == 0 ? c : c - sub_lo;
    const u32 per_set = (1u << ml) + 2 * (1u << mh);
    const XYZZ* src = rc + (size_t)set * per_set + (kind == 0 ? 0 : (1u << ml));
    const u32 cnt = 1u << (kind ? mh : ml);
    const u32 qid = threadIdx.x >> 2;
    XYZZ w = XYZZ::identity();
    for (u32 j = sub * WQ + qid; j < cnt && j < (sub + 1) * WQ; j += 64) quad_add_nl(w, XYZZ::load(src + j));
    w = quad_block_sum(w, sh);
    if (threadIdx.x == 0) w.store(parts + (size_t)set * cta_per_set + c);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(done + msm, 1u) == nsets * cta_per_set - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();

    for (u32 s0 = 0; s0 < nsets; s0++) {
        // two quads add the CTA partials of S_lo and S_hi of this set
        if (qid < 2) {
            const XYZZ* p = parts + (size_t)(msm * nsets + s0) * cta_per_set + (qid == 0 ? 0 : sub_lo);
            const u32 cnt = qid == 0 ? sub_lo : sub_hi;
            XYZZ a = XYZZ::load(p);
            for (u32 i = 1; i < cnt; i++) quad_add_nl(a, XYZZ::load(p + i));
            if ((threadIdx.x & 3) == 0) a.store(comb + qid);
        }
        __syncthreads();
        if (qid == 0) {
            XYZZ v = XYZZ::load(comb + 0);
            quad_add_nl(v, XYZZ::load(comb + 1));
            if (threadIdx.x == 0) v.store(vsets + s0);
        }
        __syncthreads();
    }
    if (qid == 0) {
        XYZZ total = XYZZ::load(vsets + nsets - 1);
        for (int s2 = (int)nsets - 2; s2 >= 0; s2--) {
            for (int d = 0; d < shift; d++) quad_dbl_nl(total);
            quad_add_nl(total, XYZZ::load(vsets + s2));
        }
        if (threadIdx.x == 0) {
            store_jacobian(total, (char*)out + 96 * (size_t)msm);
            done[msm] = 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------ SRS table
// next[i] = 2^c * prev[i], normalised to affine (one inversion per point; runs once per SRS upload)
__global__ void __launch_bounds__(128) k_precompute_level(const Affine* __restrict__ prev, Affine* __restrict__ next,
                                                          u32 count, int c) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Affine a = Affine::load(prev + i);
    if (a.is_identity()) {
        a.store(next + i);
        return;
    }
    XYZZ p = xyzz_dbl_affine(a);
    for (int d = 1; d < c; d++) p = xyzz_dbl(p);
    xyzz_to_affine(p).store(next + i);
}

// ------------------------------------------------------------------------------------------------ small group ops
__global__ void __launch_bounds__(256) k_g1_sum(const uint64_t* __restrict__ pts, u32 m, void* __restrict__ out) {
    __shared__ XYZZ sh[8];
    const u32 qid = threadIdx.x >> 2;
    XYZZ acc = XYZZ::identity();
    for (u32 i = qid; i < m; i += 64) quad_add_nl(acc, xyzz_from_jacobian(pts + 12 * (size_t)i));
    XYZZ r = quad_block_sum(acc, sh);
    if (threadIdx.x == 0) store_jacobian(r, out);
}
__global__ void __launch_bounds__(128) k_g1_normalize(uint64_t* __restrict__ pts, u32 m) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    XYZZ p = xyzz_from_jacobian(pts + 12 * (size_t)i);
    xyzz_store_jacobian_normalised(p, pts + 12 * (size_t)i);
}
// out[i] = s_i * base: plain double-and-add over the canonical scalar bits (setup-side utility)
__global__ void __launch_bounds__(128) k_fixed_base_mul(Affine base, const uint64_t* __restrict__ scalars, u32 n,
                                                        Affine* __restrict__ out) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = Fr::load_nc(scalars + 4 * (size_t)i).from_mont();
    XYZZ acc = XYZZ::identity();
    for (int limb = 7; limb >= 0; limb--) {
        u32 v = 0;
#pragma unroll
        for (int t = 0; t < 8; t++)
            if (t == limb) v = s.l[t];
        for (int bit = 31; bit >= 0; bit--) {
            acc = xyzz_dbl(acc);
            if ((v >> bit) & 1) xyzz_madd(acc, base);
        }
    }
    xyzz_to_affine(acc).store(out + i);
}

template <class F>
__global__ void __launch_bounds__(128) k_field_op(int op, const uint64_t* __restrict__ a,
                                                  const uint64_t* __restrict__ b, u32 n, uint64_t* __restrict__ out) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    F x = F::load(a + 4 * (size_t)i), y = F::zero(), r;
    if (op <= 2 || op == 7 || op == 8 || op == 10) y = F::load(b + 4 * (size_t)i);
    switch (op) {
        case 0: r = x * y; break;
        case 1: r = x + y; break;
        case 2: r = x - y; break;
        case 3: r = x.inv(); break;
        case 4: r = x.from_mont(); break;
        case 6: r = x.sqr(); break;
        case 7: r = F::mul_add_mul(x, y, x + y, x - y); break;  // a*b + (a+b)(a-b)
        case 8: r = F::mul_sub_mul(x, y, y, y); break;          // a*b - b*b
        case 9: r = x.inv_bgcd(); break;
        case 10:  // a*b + c*d on four independent operands: the second pair sits n elements further on
            r = F::mul_add_mul(x, y, F::load(a + 4 * ((size_t)n + i)), F::load(b + 4 * ((size_t)n + i)));
            break;
        default: r = x.to_mont(); break;
    }
    r.store(out + 4 * (size_t)i);
}

// ------------------------------------------------------------------------------------------------ host side
int msm_choose_c_fixed(size_t n) {
    // one bucket set of 2^(c-1) buckets, ceil(255/c) table levels: cost ~ 10*n*W + 32*2^(c-1) field mults
    // W = ceil(255 / c) only drops at c = 13, 14, 15, 16, 17, 19, 20, 22, so only those are candidates (a sweep edits the
    // constants below and rebuilds): the bucket-side work grows 2^c while the additions only shrink with W.  Small
    // domains — the shards of a multi-GPU run and the k <= 16 configs — want c close to log2(n): the fixed tail is
    // latency-bound and hardly grows with the bucket count, while fewer table levels shorten everything else.
    // Measured on an H100 80GB HBM3 at a 400 W power limit (one MSM, uniform / witness-like scalars): 2^19: c = 17
    // 23.6 ms per k = 19 bench step against 24.0 (16), 27.4 (19), 27.8 (20); 2^21: c = 17 7.16 / 2.61 ms against
    // 7.35 / 3.19 ms at c = 20; 2^23: c = 20 27.1 / 9.0 ms against 30.6 / 9.1 at c = 17.  2^22 is not measured.
    const int lg = ceil_log2(n ? n : 1);
    if (lg >= 22) return 20;
    if (lg >= 17) return 17;
    if (lg == 16) return 16;
    if (lg >= 13) return 15;
    if (lg >= 11) return 13;
    return lg < 8 ? 8 : lg;
}
static int msm_choose_c_adhoc(size_t n) {
    int lg = ceil_log2(n ? n : 1);
    int c = lg - 4;
    if (c < 6) c = 6;
    if (c > 16) c = 16;
    return c;
}

void msm_build_table(h2b_ctx* ctx, const void* d_bases, size_t count, int c, int W, void* d_table) {
    Affine* t = reinterpret_cast<Affine*>(d_table);
    H2B_CUDA(cudaMemcpyAsync(t, d_bases, count * sizeof(Affine), cudaMemcpyDeviceToDevice, ctx->stream));
    for (int w = 1; w < W; w++)
        H2B_LAUNCH(ctx, k_precompute_level, ceil_div(count, 128), 128, 0, t + (size_t)(w - 1) * count,
                   t + (size_t)w * count, (u32)count, c);
}

// m MSMs of the same size through one pipeline (table mode: q == W, one bucket set per MSM; ad-hoc mode: m == 1).
// The m results are stored at d_out + 96 * j.
void msm_run_group(h2b_ctx* ctx, const void* const* d_tables, size_t n, int c, int W, int q, const void* const* d_scalars, size_t m,
                   void* d_out, cudaEvent_t after_digits) {
    H2B_REQUIRE(n >= 1 && n <= ((size_t)1 << 27), "msm: n out of range");
    H2B_REQUIRE((size_t)W * n < ((size_t)1 << 31) - 8, "msm: n * windows exceeds the 31-bit table index");
    H2B_REQUIRE(m >= 1 && m <= (size_t)MSM_MAX_GROUP, "msm: group size out of range");
    H2B_REQUIRE(m == 1 || q == W, "msm: groups need tabulated bases");
    const u32 nbw = 1u << (c - 1);
    const u32 nsets = (u32)((W + q - 1) / q);  // bucket sets of one MSM
    const u32 nb_group = nsets * nbw;          // buckets of one MSM
    const u32 nb_total = (u32)m * nb_group;
    const size_t M = (size_t)W * n * m;
    cudaStream_t st = ctx->stream;
    H2B_REQUIRE(M < ((size_t)1 << 32), "msm: entry count exceeds 32 bits");
    MsmScalars cols;
    const Affine* tab_a = (const Affine*)d_tables[0];
    const Affine* tab_b = tab_a;
    u32 table_mask = 0;  // bit j: MSM j reads the second table
    for (size_t j = 0; j < (size_t)MSM_MAX_GROUP; j++) cols.p[j] = (const uint64_t*)d_scalars[j < m ? j : 0];
    for (size_t j = 1; j < m; j++) {
        if (d_tables[j] == (const void*)tab_a) continue;
        if (tab_b == tab_a) tab_b = (const Affine*)d_tables[j];
        H2B_REQUIRE(d_tables[j] == (const void*)tab_b, "msm: a group reads at most two distinct tables");
        table_mask |= 1u << j;
    }
    H2B_REQUIRE(table_mask == 0 || (size_t)W * n < ((size_t)1 << 30), "msm: two-table groups need n * windows < 2^30");

    // coarse bins of the sort: key >> F.  About 256 bins: a partition tile (256 scalars x W digits) then writes runs of ~15
    // entries per bin, and a bin's 2^F buckets are counted in shared memory by the fine passes.
    int F = 0;
    while (F < SORT_F_MAX && (((size_t)nb_total + (1u << F) - 1) >> F) > 256) F++;
    const u32 nbins = (u32)(((size_t)nb_total + (1u << F) - 1) >> F);
    H2B_REQUIRE(nbins <= (u32)SORT_BINS_MAX, "msm: too many buckets for the sort");
    const size_t part_smem = 2 * (size_t)nbins * 4 + (size_t)W * SORT_PART_TS * 12;
    H2B_REQUIRE(part_smem <= (size_t)SORT_PART_SMEM_MAX, "msm: too many windows for the sort");
    if (!ctx->sort_attr_set) {  // per context: the attribute belongs to the device the context is bound to
        H2B_CUDA(cudaFuncSetAttribute(k_sort_partition, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_PART_SMEM_MAX));
        H2B_CUDA(cudaFuncSetAttribute(k_sort_fine<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_FINE_SMEM));
        ctx->sort_attr_set = true;
    }

    u32* vals = (u32*)ctx->get(WS_VALS_A, M * 4 + 16);  // W * n * m: room for every digit, zero or not
    // the partitioned entries: low key bits and sorted-entry value, 6 bytes per non-zero digit
    uint16_t* tmp_low = (uint16_t*)ctx->get(WS_KEYS_B, M * 2 + 16);
    u32* tmp_val = (u32*)ctx->get(WS_VALS_B, M * 4 + 16);
    const u32 ntiles = (nb_total + SCAN_TILE - 1) / SCAN_TILE;
    // bin counts and bucket histogram (zeroed together; hist[nb_total] counts the finished CTAs of k_sort_count), cursors,
    // scan tile sums, L, bin bases, bin cursors, chunk prefix
    u32* cnt = (u32*)ctx->get(WS_KEYS_A, (2 * ((size_t)nb_total + 2) + ntiles + 4 * (size_t)nbins + 8) * 4);
    u32* bin_count = cnt;
    u32* hist = bin_count + nbins;
    u32* cursor = hist + nb_total + 2;
    u32* tile_sums = cursor + nb_total + 2;
    u32* d_L = tile_sums + ntiles + 1;
    u32* bin_base = d_L + 1;
    u32* bin_cursor = bin_base + nbins + 1;
    u32* chunk_pre = bin_cursor + nbins;
    u32* off = (u32*)ctx->get(WS_OFFSETS, ((size_t)nb_total + 2) * 4);
    XYZZ* buckets = (XYZZ*)ctx->get(WS_BUCKETS, (size_t)nb_total * sizeof(XYZZ));
    const u32 l_min = 12u, l_max = (u32)ACC_L_DEFAULT;  // chunk length of k_accumulate, chosen on the device in [12, 32]
    const u32 slots = (u32)ctx->sm_count * 512u;  // k_accumulate: 128 registers -> 4 CTAs x 128 threads per SM
    // chunks of k_accumulate: L < l_max is only chosen when the entries do not fill one wave, i.e. at most `slots` chunks
    const size_t n_chunks = std::max((M + l_max - 1) / l_max, (size_t)slots) + 1;
    XYZZ* partials = (XYZZ*)ctx->get(WS_PARTIALS, 2 * n_chunks * sizeof(XYZZ));
    u32* big = (u32*)ctx->get(WS_BIGLIST, ((size_t)nb_total + 1) * 4);  // [0] = counter, list follows

    // two-level sort by bucket (see k_sort_count): digits are recomputed from the scalars, not stored
    H2B_CUDA(cudaMemsetAsync(cnt, 0, ((size_t)nbins + nb_total + 1) * 4, st));
    // the keys of all digits ([msm][window][scalar], NO_DIGIT for a zero digit) live in `vals` until k_sort_fine<1> overwrites it
    u32* keys = vals;
    H2B_LAUNCH(ctx, k_sort_count, dim3(ceil_div(n, 256), (unsigned)m), 256, 0, cols, (u32)n, c, W, q, nbw, nsets, F, nbins,
               bin_count, keys, hist + nb_total, bin_base, bin_cursor, chunk_pre);
    if (after_digits) H2B_CUDA(cudaEventRecord(after_digits, st));  // the scalars are not read after this point
    H2B_LAUNCH(ctx, k_sort_partition, dim3(ceil_div(n, SORT_PART_TS), (unsigned)m), SORT_PART_TS, part_smem, keys, (u32)n, W, q,
               nbw, table_mask, F, nbins, bin_cursor, tmp_low, tmp_val);
    const unsigned fine_grid = ceil_div(M, SORT_CHUNK) + nbins;  // chunks of all bins together: at most this many
    H2B_LAUNCH(ctx, k_sort_fine<0>, fine_grid, 512, (size_t)4 << F, chunk_pre, bin_base, nbins, F, tmp_low, tmp_val, hist,
               (u32*)nullptr);
    H2B_LAUNCH(ctx, k_scan_tiles, ntiles, 256, 0, hist, nb_total, off, tile_sums);
    H2B_LAUNCH(ctx, k_scan_apply, ntiles, 256, 0, nb_total, ntiles, tile_sums, off, cursor, slots, l_min, l_max, d_L);
    H2B_LAUNCH(ctx, k_sort_fine<1>, fine_grid, 512, ((size_t)8 << F) + SORT_CHUNK * 6, chunk_pre, bin_base, nbins, F, tmp_low,
               tmp_val, cursor, vals);

    H2B_CUDA(cudaMemsetAsync(big, 0, 4, st));
    H2B_LAUNCH(ctx, k_accumulate, ceil_div(n_chunks, 128), 128, 0, vals, off, nb_total, d_L, tab_a, tab_b, buckets, partials);
    // From here on the work is a few hundred CTAs of dependent point additions.  Inside a lane (other MSMs of the batch are
    // in flight on the other lanes) it moves to the lane's high-priority stream: the block scheduler hands freed SM slots to
    // it before the queued accumulation waves of the next MSM, so the latency-bound tail overlaps that accumulation instead
    // of waiting for it to drain.  The lane stream waits for the tail (same order for the caller, workspaces stay safe).
    const bool tail_hp = ctx->in_lane;
    struct TailScope {  // restores the lane stream and makes it wait for the tail on every exit path
        h2b_ctx* c; cudaStream_t lane; bool on;
        ~TailScope() {
            if (!on) return;
            cudaEventRecord(c->lane_tail_done[c->cur_lane], c->stream);
            c->stream = lane;
            cudaStreamWaitEvent(lane, c->lane_tail_done[c->cur_lane], 0);
        }
    } tail_scope{ctx, st, tail_hp};
    if (tail_hp) {
        H2B_CUDA(cudaEventRecord(ctx->lane_acc[ctx->cur_lane], st));
        ctx->stream = ctx->lane_tail[ctx->cur_lane];
        H2B_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->lane_acc[ctx->cur_lane], 0));
    }
    H2B_LAUNCH(ctx, k_collect, ceil_div(nb_total, 128), 128, 0, off, nb_total, d_L, partials, buckets, big + 1, big);
    XYZZ* seg = (XYZZ*)ctx->get(WS_POOL, (2 * (n_chunks / BIG_SEG) + 64) * sizeof(XYZZ));
    H2B_LAUNCH(ctx, k_collect_big1, 2 * ctx->sm_count, 256, 0, off, d_L, partials, big + 1, big, seg);
    H2B_LAUNCH(ctx, k_collect_big2, 64, 256, 0, off, d_L, seg, buckets, big + 1, big);

    // bucket reduction: row/column sums of the 2^mh x 2^ml bucket grid, small scalar multiples, final combine
    const int mm = c - 1, ml = (mm + 1) / 2, mh = mm - ml;
    H2B_REQUIRE(nsets <= 64, "msm: too many bucket sets");
    const u32 all_sets = nsets * (u32)m;
    const u32 per_set = (1u << ml) + (1u << mh);  // row + column sums (one CTA each)
    const u32 sub_lo = ((1u << ml) + WQ - 1) / WQ, sub_hi = ((1u << mh) + WQ - 1) / WQ;
    const u32 cta_per_set = sub_lo + sub_hi;
    XYZZ* rc = (XYZZ*)ctx->get(WS_REDUCE_A, (size_t)all_sets * (per_set + (1u << mh)) * sizeof(XYZZ));
    char* rb = (char*)ctx->get(WS_REDUCE_B, (size_t)all_sets * cta_per_set * sizeof(XYZZ) + 256);
    XYZZ* parts = (XYZZ*)rb;
    u32* done = (u32*)(rb + (size_t)all_sets * cta_per_set * sizeof(XYZZ));  // one counter per MSM of the group
    H2B_CUDA(cudaMemsetAsync(done, 0, 4 * MSM_MAX_GROUP, ctx->stream));
    H2B_LAUNCH(ctx, k_rowcol_sums, all_sets * per_set, 128, 0, buckets, ml, mh, all_sets, rc);
    H2B_LAUNCH(ctx, k_rowcol_weights, ceil_div((size_t)all_sets * per_set * 4, 128), 128, 0, rc, ml, mh, all_sets);
    H2B_LAUNCH(ctx, k_weighted_final, all_sets * cta_per_set, 256, 0, rc, ml, mh, nsets, c * q, parts, done, d_out);
}

void msm_run(h2b_ctx* ctx, const void* d_table, size_t n, int c, int W, int q, const void* d_scalars, void* d_out,
             cudaEvent_t after_digits) {
    msm_run_group(ctx, &d_table, n, c, W, q, &d_scalars, 1, d_out, after_digits);
}

void g1_sum_run(h2b_ctx* ctx, const void* d_points, size_t m, void* d_out) {
    H2B_LAUNCH(ctx, k_g1_sum, 1, 256, 0, (const uint64_t*)d_points, (u32)m, d_out);
}
void g1_normalize_run(h2b_ctx* ctx, void* d_points, size_t m) {
    if (m == 0) return;
    H2B_LAUNCH(ctx, k_g1_normalize, ceil_div(m, 128), 128, 0, (uint64_t*)d_points, (u32)m);
}
void g1_fixed_base_mul_run(h2b_ctx* ctx, const uint64_t base_xy[8], const void* d_scalars, size_t n, void* d_out) {
    if (n == 0) return;
    Affine b;
    memcpy(&b, base_xy, sizeof(Affine));
    H2B_LAUNCH(ctx, k_fixed_base_mul, ceil_div(n, 128), 128, 0, b, (const uint64_t*)d_scalars, (u32)n, (Affine*)d_out);
}
void field_op_run(h2b_ctx* ctx, int field, int op, const void* a, const void* b, size_t n, void* out) {
    if (n == 0) return;
    if (field == 0)
        H2B_LAUNCH(ctx, k_field_op<Fq>, ceil_div(n, 128), 128, 0, op, (const uint64_t*)a, (const uint64_t*)b, (u32)n, (uint64_t*)out);
    else
        H2B_LAUNCH(ctx, k_field_op<Fr>, ceil_div(n, 128), 128, 0, op, (const uint64_t*)a, (const uint64_t*)b, (u32)n, (uint64_t*)out);
}

// Runs `fn(lane)` with the context switched to lane `lane` (its stream and workspace set).
struct LaneScope {
    h2b_ctx* ctx;
    cudaStream_t saved_stream;
    int saved_lane;
    LaneScope(h2b_ctx* c, int lane) : ctx(c), saved_stream(c->stream), saved_lane(c->cur_lane) {
        c->stream = c->lane_stream[lane];
        c->cur_lane = lane;
        c->in_lane = true;
    }
    ~LaneScope() {
        ctx->stream = saved_stream;
        ctx->cur_lane = saved_lane;
        ctx->in_lane = false;
    }
};

// How many MSMs of a batch share one pipeline (msm_run_group).  Large domains: the accumulation dominates and lanes of
// single MSMs overlap one MSM's sort / tail with the next one's accumulation; small domains (k <= 17, the shards of a
// multi-GPU run) are bound by the latency of the bucket reduction, which a group pays once.
size_t msm_group_size(const h2b_ctx* ctx, size_t n, size_t m, int W) {
    if ((size_t)W * n >= ((size_t)1 << 30)) return 1;  // no room for the table bit in a sorted entry: one MSM per pipeline
    size_t g = ctx->opt_msm_group > 0 ? (size_t)ctx->opt_msm_group : 0;
    if (g == 0) {
        const int lg = ceil_log2(n);
        g = lg <= 17 ? MSM_MAX_GROUP : (lg <= 19 ? (m + 1) / 2 : (m + 2) / 3);
    }
    if (g > (size_t)MSM_MAX_GROUP) g = MSM_MAX_GROUP;
    while (g > 1 && g * (size_t)W * n >= ((size_t)1 << 32)) g--;  // sorted positions are 32-bit
    return g < 1 ? 1 : g;
}

void msm_run_batch(h2b_ctx* ctx, const void* const* d_tables, size_t n, int c, int W, const void* const* d_scalars, size_t m,
                   void* d_out) {
    if (m == 0) return;
    const size_t gsz = msm_group_size(ctx, n, m, W);
    const size_t ngroups = (m + gsz - 1) / gsz;
    if (ngroups == 1) {  // nothing to overlap: stay on the caller's stream
        msm_run_group(ctx, d_tables, n, c, W, W, d_scalars, m, d_out, nullptr);
        return;
    }
    cudaStream_t main = ctx->stream;
    H2B_CUDA(cudaEventRecord(ctx->fork_ev, main));
    const int nl = (int)(ngroups < (size_t)h2b_ctx::NLANES ? ngroups : (size_t)h2b_ctx::NLANES);
    for (int l = 0; l < nl; l++) H2B_CUDA(cudaStreamWaitEvent(ctx->lane_stream[l], ctx->fork_ev, 0));
    struct Join {  // the lanes are joined back onto the caller's stream on every exit path (a throw included)
        h2b_ctx* c; cudaStream_t main; int nl;
        ~Join() {
            for (int l = 0; l < nl; l++) {
                cudaEventRecord(c->lane_done[l], c->lane_stream[l]);
                cudaStreamWaitEvent(main, c->lane_done[l], 0);
            }
        }
    } join{ctx, main, nl};
    // balanced groups (sizes differ by at most one), dealt to the lanes round-robin
    size_t j = 0;
    for (size_t g = 0; g < ngroups; g++) {
        const size_t cnt = m / ngroups + (g < m % ngroups ? 1 : 0);
        LaneScope scope(ctx, (int)(g % nl));
        msm_run_group(ctx, d_tables + j, n, c, W, W, d_scalars + j, cnt, (char*)d_out + 96 * j, nullptr);
        j += cnt;
    }
}

// ad-hoc bases: W bucket sets, no table
void msm_run_adhoc(h2b_ctx* ctx, const void* d_bases, size_t n, const void* d_scalars, void* d_out) {
    int c = msm_choose_c_adhoc(n);
    int W = (255 + c - 1) / c;
    msm_run(ctx, d_bases, n, c, W, 1, d_scalars, d_out);
}

}  // namespace h2b
