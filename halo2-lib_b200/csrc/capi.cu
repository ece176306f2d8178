// capi.cu — the extern "C" surface declared in include/h2b200.h: context, SRS handles, staging of host buffers.
// No exception leaves this file: every entry point maps failures to a status code + h2b_last_error().
#include <cstring>
#include <functional>

#include "h2b_internal.cuh"

namespace h2b {
void msm_run_adhoc(h2b_ctx* ctx, const void* d_bases, size_t n, const void* d_scalars, void* d_out);
static std::string g_create_error;
static std::mutex g_create_mu;
}  // namespace h2b

using namespace h2b;

void* h2b_ctx::get(int slot, size_t bytes) {
    if (bytes == 0) bytes = 16;
    Buf& b = ws[cur_lane][slot];
    if (b.cap >= bytes) return b.p;
    if (b.p) {
        H2B_CUDA(cudaDeviceSynchronize());
        cudaFree(b.p);
        b.p = nullptr;
        b.cap = 0;
    }
    size_t cap = bytes + bytes / 8;
    cap = (cap + 255) & ~(size_t)255;
    H2B_CUDA(cudaMalloc(&b.p, cap));
    b.cap = cap;
    return b.p;
}
void* h2b_ctx::get_pinned(int slot, size_t bytes) {
    if (bytes == 0) bytes = 16;
    Buf& b = pinned[slot];
    if (b.cap >= bytes) return b.p;
    if (b.p) {
        H2B_CUDA(cudaDeviceSynchronize());
        cudaFreeHost(b.p);
        b.p = nullptr;
        b.cap = 0;
    }
    H2B_CUDA(cudaMallocHost(&b.p, bytes));
    b.cap = bytes;
    return b.p;
}

cudaEvent_t h2b_ctx::prof_event() {
    if (!prof_pool.empty()) {
        cudaEvent_t e = prof_pool.back();
        prof_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    H2B_CUDA(cudaEventCreate(&e));
    return e;
}

// ---- device group helpers (h2b_ctx_create_multi): run `fn(member, index)` with the member's device current
template <class Fn>
static void group_each(h2b_ctx* ctx, Fn&& fn) {
    for (size_t i = 0; i < ctx->members.size(); i++) {
        H2B_CUDA(cudaSetDevice(ctx->members[i]->device));
        fn(ctx->members[i], i);
    }
    H2B_CUDA(cudaSetDevice(ctx->device));
}
template <class T>
static std::vector<T> every_gth(T const* v, size_t m, size_t g, size_t G) {
    std::vector<T> r;
    for (size_t j = g; j < m; j += G) r.push_back(v[j]);
    return r;
}

// The staging of a host-pointer entry point, which is its `_dev` form run on copies of the host buffers: one ctx->get of
// `bytes` in `slot` (the slot keeps the copies apart from the scratch the `*_run` function takes), carved into the
// inputs, scratch and outputs of the call.  Uploads are enqueued on ctx->stream as the regions are carved; finish()
// enqueues the downloads of the output regions and synchronises once.
namespace {
struct Staging {
    struct Download {
        void* host;
        const void* dev;
        size_t bytes;
    };
    h2b_ctx* ctx;
    char* base;
    size_t used = 0, cap;
    std::vector<Download> downloads;
    Staging(h2b_ctx* c, int slot, size_t bytes) : ctx(c), cap(bytes) { base = (char*)c->get(slot, bytes); }
    // the next `bytes` of the slot, 32-byte aligned
    char* take(size_t bytes) {
        const size_t at = (used + 31) & ~(size_t)31;
        H2B_REQUIRE(at + bytes <= cap, "staging overflow");
        used = at + bytes;
        return base + at;
    }
    // an input: `bytes` from the host, uploaded into the next `room` (at least `bytes`) bytes of the slot
    char* up(const void* host, size_t bytes, size_t room = 0) {
        char* d = take(room > bytes ? room : bytes);
        if (bytes) H2B_CUDA(cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
        return d;
    }
    // an output: the first `bytes` of the next `room` (at least `bytes`) bytes go to `host` (nowhere when it is null)
    char* out(void* host, size_t bytes, size_t room = 0) {
        char* d = take(room > bytes ? room : bytes);
        if (host && bytes) downloads.push_back({host, d, bytes});
        return d;
    }
    // an input that is also the output
    char* inout(void* host, size_t bytes) {
        char* d = up(host, bytes);
        if (bytes) downloads.push_back({host, d, bytes});
        return d;
    }
    void finish() {
        for (auto& x : downloads) H2B_CUDA(cudaMemcpyAsync(x.host, x.dev, x.bytes, cudaMemcpyDeviceToHost, ctx->stream));
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    }
};
}  // namespace

// Every stream and event a context owns, in one list that h2b_ctx_create creates and h2b_ctx_destroy destroys.  Three
// stream priority levels.  Highest: the bucket reduction of a lane's MSM — its few CTAs take the SM slots that free up
// first instead of queueing behind the next MSM's accumulation waves (see msm_run_group).  Middle: the lanes and the
// context's own stream.  Lowest (the default of a plain stream): the copy streams, the side queue and whatever else the
// caller runs beside the commitments — the polynomial transforms fill the bubbles the MSM pipeline leaves.
enum StreamPrio { PRIO_DEFAULT, PRIO_LANE, PRIO_TAIL };
template <class Stream, class Event>
static void ctx_handles(h2b_ctx* ctx, Stream&& stream, Event&& event) {
    stream(ctx->own_stream, PRIO_LANE);
    stream(ctx->copy_stream, PRIO_DEFAULT);
    stream(ctx->copy_stream2, PRIO_DEFAULT);
    stream(ctx->side_stream, PRIO_DEFAULT);
    for (auto& e : ctx->side_ev) event(e);
    for (auto& row : ctx->pipe_ev)
        for (auto& e : row) event(e);
    for (auto& e : ctx->ev) event(e);
    for (int l = 0; l < h2b_ctx::NLANES; l++) {
        stream(ctx->lane_stream[l], PRIO_LANE);
        stream(ctx->lane_tail[l], PRIO_TAIL);
        event(ctx->lane_acc[l]);
        event(ctx->lane_tail_done[l]);
        event(ctx->lane_done[l]);
        event(ctx->lane_ready[l]);
        event(ctx->lane_consumed[l]);
    }
    event(ctx->fork_ev);
}
static void destroy_handles(h2b_ctx* ctx) {
    ctx_handles(ctx, [](cudaStream_t& s, StreamPrio) { if (s) cudaStreamDestroy(s); }, [](cudaEvent_t& e) { if (e) cudaEventDestroy(e); });
}

// m columns through three rotating buffer sets: the upload of column i+1 (copy stream) and the downloads of column i-1
// (second copy stream) overlap the kernels of column i (context stream).  Column i uses set b = i mod 3: it is uploaded
// from in[i] into up_buf[b], `compute(i, b)` enqueues its kernels, and `download(i, b, down)` waits for pipe_ev[b][1]
// (or an earlier event of the context stream) before each copy it enqueues.  Enqueue only: see ntt_batch_finish.
template <class Compute, class Download>
static void ntt_pipeline(h2b_ctx* ctx, const uint64_t* const* in, size_t m, void* const up_buf[3], size_t up_bytes, Compute&& compute,
                         Download&& download) {
    cudaStream_t up = ctx->copy_stream, ks = ctx->stream, down = ctx->copy_stream2;
    H2B_CUDA(cudaEventRecord(ctx->fork_ev, ks));
    H2B_CUDA(cudaStreamWaitEvent(up, ctx->fork_ev, 0));
    for (size_t i = 0; i < m; i++) {
        const int b = (int)(i % 3);
        if (i >= 3) H2B_CUDA(cudaStreamWaitEvent(up, ctx->pipe_ev[b][2], 0));  // buffer set b downloaded
        H2B_CUDA(cudaMemcpyAsync(up_buf[b], in[i], up_bytes, cudaMemcpyHostToDevice, up));
        H2B_CUDA(cudaEventRecord(ctx->pipe_ev[b][0], up));
        H2B_CUDA(cudaStreamWaitEvent(ks, ctx->pipe_ev[b][0], 0));
        compute(i, b);
        H2B_CUDA(cudaEventRecord(ctx->pipe_ev[b][1], ks));
        download(i, b, down);
        H2B_CUDA(cudaEventRecord(ctx->pipe_ev[b][2], down));
    }
}
static void ntt_batch_finish(h2b_ctx* ctx) {
    H2B_CUDA(cudaStreamSynchronize(ctx->copy_stream2));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
}
// One batch per device: on a device group (h2b_ctx_create_multi) polynomial j goes to device j mod G ("one column
// polynomial per device", SURVEY.md §8e), and every device's pipeline is enqueued before the first wait.
template <class In, class Out, class Batch>
static void ntt_deal(h2b_ctx* ctx, In const* in, Out const* out, size_t m, Batch&& batch) {
    if (ctx->members.size() <= 1) {
        batch(ctx, in, out, m);
        return ntt_batch_finish(ctx);
    }
    const size_t G = ctx->members.size();
    group_each(ctx, [&](h2b_ctx* mb, size_t g) {
        auto vi = every_gth(in, m, g, G);
        auto vo = every_gth(out, m, g, G);
        batch(mb, vi.data(), vo.data(), vi.size());
    });
    group_each(ctx, [&](h2b_ctx* mb, size_t) { ntt_batch_finish(mb); });
}

extern "C" {

const char* h2b_version(void) { return "h2b200 0.1.0 (sm_90a)"; }

int h2b_ctx_create(int device, h2b_ctx** out) {
    if (!out) return H2B_ERR_ARG;
    *out = nullptr;
    std::lock_guard<std::mutex> lock(g_create_mu);
    h2b_ctx* ctx = nullptr;
    int rc = H2B_OK;
    try {
        int ndev = 0;
        cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || ndev == 0)
            throw StatusError{H2B_ERR_CUDA, std::string("no CUDA device available (there is no CPU fallback): ") +
                                                (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0")};
        if (device < 0 || device >= ndev) throw StatusError{H2B_ERR_ARG, "device index out of range"};
        H2B_CUDA(cudaSetDevice(device));
        ctx = new h2b_ctx();
        ctx->device = device;
        int lo_prio = 0, hi_prio = 0;
        H2B_CUDA(cudaDeviceGetStreamPriorityRange(&lo_prio, &hi_prio));
        ctx_handles(ctx, [&](cudaStream_t& s, StreamPrio p) {
            if (p == PRIO_DEFAULT) H2B_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
            else H2B_CUDA(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, p == PRIO_LANE ? (lo_prio + hi_prio) / 2 : hi_prio));
        }, [](cudaEvent_t& e) { H2B_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); });
        ctx->stream = ctx->own_stream;
        cudaDeviceProp prop;
        H2B_CUDA(cudaGetDeviceProperties(&prop, device));
        ctx->sm_count = prop.multiProcessorCount;
        *out = ctx;
        return H2B_OK;
    } catch (const StatusError& e) {
        g_create_error = e.msg;
        rc = e.code;
    } catch (...) {
        g_create_error = "unknown failure in h2b_ctx_create";
        rc = H2B_ERR_CUDA;
    }
    if (ctx) destroy_handles(ctx);  // the streams and events created before the failure
    delete ctx;
    return rc;
}

// One process, several GPUs (SURVEY.md §8(b): h2b_ctx_create(const int* dev_ids, int n_dev, ...)): the returned handle is
// an ordinary context on dev_ids[0] that additionally owns one private context per further device.  h2b_srs_upload shards
// the bases over the devices by contiguous index range, the host-pointer MSM entry points commit every shard on its own
// device and combine the partial sums with the fused all-reduce kernel over in-process peer mappings (no IPC, no NCCL),
// the batched transform entry points deal the polynomials round-robin.  Everything else runs on dev_ids[0].
int h2b_ctx_create_multi(const int* dev_ids, int n_dev, h2b_ctx** out) {
    if (!out || !dev_ids || n_dev < 1 || n_dev > 16) return H2B_ERR_ARG;
    *out = nullptr;
    std::vector<h2b_ctx*> made;
    int rc = H2B_OK;
    for (int i = 0; i < n_dev && rc == H2B_OK; i++) {
        if (std::find(dev_ids, dev_ids + i, dev_ids[i]) != dev_ids + i) {
            std::lock_guard<std::mutex> lock(g_create_mu);
            g_create_error = "ctx_create_multi: duplicate device id";
            rc = H2B_ERR_ARG;
        } else {
            h2b_ctx* c = nullptr;
            rc = h2b_ctx_create(dev_ids[i], &c);  // on failure it has set the message
            if (rc == H2B_OK) made.push_back(c);
        }
    }
    if (rc == H2B_OK) {
        made[0]->members = made;
        if (n_dev > 1 && (rc = guarded(made[0], [&] { peer_connect_local(made); })) != H2B_OK) {
            std::lock_guard<std::mutex> lock(g_create_mu);
            g_create_error = made[0]->err;
            made[0]->members.clear();  // every context is destroyed on its own below
        }
    }
    if (rc != H2B_OK) {
        for (auto* m : made) h2b_ctx_destroy(m);
        return rc;
    }
    *out = made[0];
    return H2B_OK;
}
int h2b_ctx_device_count(const h2b_ctx* ctx) { return ctx ? (int)(ctx->members.empty() ? 1 : ctx->members.size()) : 0; }

void h2b_ctx_destroy(h2b_ctx* ctx) {
    if (!ctx) return;
    if (ctx->members.size() > 1) {  // a device group: the private member contexts go first
        std::vector<h2b_ctx*> others(ctx->members.begin() + 1, ctx->members.end());
        ctx->members.clear();
        for (auto* m : others) h2b_ctx_destroy(m);
    }
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    ntt_free_plans(ctx);
    peer_destroy(ctx);
    for (auto& lane : ctx->ws)
        for (auto& b : lane)
            if (b.p) cudaFree(b.p);
    for (auto& b : ctx->pinned)
        if (b.p) cudaFreeHost(b.p);
    for (auto& r : ctx->prof_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (auto& e : ctx->prof_pool) cudaEventDestroy(e);
    destroy_handles(ctx);
    delete ctx;
}

int h2b_ctx_set_stream(h2b_ctx* ctx, void* cuda_stream) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(!ctx->side_saved, "set_stream: not while the side stream is current");
        ctx->stream = cuda_stream ? (cudaStream_t)cuda_stream : ctx->own_stream;
    });
}
int h2b_ctx_side_begin(h2b_ctx* ctx) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(!ctx->side_saved, "side_begin: the side stream is already current");
        H2B_CUDA(cudaEventRecord(ctx->side_ev[0], ctx->stream));
        H2B_CUDA(cudaStreamWaitEvent(ctx->side_stream, ctx->side_ev[0], 0));
        ctx->side_saved = ctx->stream;
        ctx->stream = ctx->side_stream;
        ctx->side_saved_lane = ctx->cur_lane;
        ctx->cur_lane = 1;  // own scratch buffers: the two queues never share a workspace slot
    });
}
int h2b_ctx_side_end(h2b_ctx* ctx) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(ctx->side_saved, "side_end: the side stream is not current");
        ctx->stream = ctx->side_saved;
        ctx->side_saved = nullptr;
        ctx->cur_lane = ctx->side_saved_lane;
    });
}
int h2b_ctx_side_join(h2b_ctx* ctx) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(!ctx->side_saved, "side_join: call h2b_ctx_side_end first");
        H2B_CUDA(cudaEventRecord(ctx->side_ev[1], ctx->side_stream));
        H2B_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->side_ev[1], 0));
    });
}
int h2b_ctx_set_option(h2b_ctx* ctx, const char* key, int64_t value) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(key, "set_option: null key");
        const std::string k(key);
        if (k == "ntt.max_ctas_per_sm") { H2B_REQUIRE(value >= 0 && value <= 2, "ntt.max_ctas_per_sm: 0 (no limit), 1 or 2"); ctx->opt_ntt_ctas = (int)value; }
        else if (k == "msm.batch_group") { H2B_REQUIRE(value >= 0 && value <= 16, "msm.batch_group: 0 (default) .. 16 MSMs per pipeline"); ctx->opt_msm_group = (int)value; }
        else if (k == "lookup.leftover_order") { H2B_REQUIRE(value == 0 || value == 1, "lookup.leftover_order: 0 (front to back) or 1 (zcash: from the back)"); ctx->opt_lookup_backward = (int)value; }
        else H2B_REQUIRE(false, "set_option: unknown key");
    });
}
int h2b_ctx_synchronize(h2b_ctx* ctx) {
    return guarded(ctx, [&] { H2B_CUDA(cudaStreamSynchronize(ctx->stream)); });
}
const char* h2b_last_error(const h2b_ctx* ctx) {
    // the message is copied under the lock into a per-thread buffer: rayon workers may fail concurrently
    static thread_local std::string tl;
    if (ctx) {
        std::lock_guard<std::mutex> lock(ctx->mu);
        tl = ctx->err;
    } else {
        std::lock_guard<std::mutex> lock(g_create_mu);
        tl = g_create_error;
    }
    return tl.c_str();
}
uint64_t h2b_kernel_launches(const h2b_ctx* ctx) {
    if (!ctx) return 0;
    uint64_t n = ctx->launches;
    for (size_t i = 1; i < ctx->members.size(); i++) n += ctx->members[i]->launches;
    return n;
}

// ------------------------------------------------------------------------------------------------ profiling
int h2b_profile_enable(h2b_ctx* ctx, const char* filter) {
    return guarded(ctx, [&] { ctx->prof_filter = filter ? filter : ""; });
}
int h2b_profile_reset(h2b_ctx* ctx) {
    return guarded(ctx, [&] {
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
        for (auto& r : ctx->prof_recs) { ctx->prof_pool.push_back(r.a); ctx->prof_pool.push_back(r.b); }
        ctx->prof_recs.clear();
    });
}
int h2b_profile_read(h2b_ctx* ctx, const char* kernel, double* total_ms, uint64_t* launches) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(kernel && total_ms && launches, "profile_read: null pointer");
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
        double ms = 0;
        uint64_t cnt = 0;
        for (auto& r : ctx->prof_recs) {
            if (std::string(r.name).find(kernel) == std::string::npos) continue;
            float t = 0;
            H2B_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
            ms += t;
            cnt++;
        }
        *total_ms = ms;
        *launches = cnt;
    });
}

// Timeline of the recorded launches: one CSV line per launch — kernel, stream, start and end in microseconds after
// `origin` (an event the caller recorded; pass the same one to several contexts of a device to align their timelines).
int h2b_profile_dump(h2b_ctx* ctx, void* origin_cuda_event, const char* path) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(origin_cuda_event && path, "profile_dump: null pointer");
        H2B_CUDA(cudaDeviceSynchronize());
        FILE* f = fopen(path, "a");
        H2B_REQUIRE(f, "profile_dump: cannot open the file");
        for (auto& r : ctx->prof_recs) {
            float a = 0, b = 0;
            if (cudaEventElapsedTime(&a, (cudaEvent_t)origin_cuda_event, r.a) != cudaSuccess ||
                cudaEventElapsedTime(&b, (cudaEvent_t)origin_cuda_event, r.b) != cudaSuccess) {
                cudaGetLastError();
                continue;
            }
            fprintf(f, "%s,%p,%.1f,%.1f\n", r.name, (void*)r.stream, a * 1e3, b * 1e3);
        }
        fclose(f);
    });
}

// ------------------------------------------------------------------------------------------------ SRS
// Frees a handle and its tables; a device group's parts each on their own device once that device is idle.  The caller
// holds the context lock.
static void srs_free(h2b_ctx* ctx, h2b_srs* s) {
    for (size_t i = 0; i < s->parts.size(); i++) {
        cudaSetDevice(ctx->members[i]->device);
        cudaDeviceSynchronize();
        for (auto& t : s->parts[i]->table)
            if (t) cudaFree(t);
        delete s->parts[i];
    }
    if (ctx) {
        cudaSetDevice(ctx->device);
        cudaDeviceSynchronize();
    }
    for (auto& t : s->table)
        if (t) cudaFree(t);
    delete s;
}

static void srs_build(h2b_ctx* ctx, const void* d_g, const void* d_gl, uint32_t k, size_t begin, size_t count, h2b_srs** out) {
    H2B_REQUIRE(out, "srs: null output handle");
    H2B_REQUIRE(k <= 27, "srs: k out of range");
    H2B_REQUIRE(count >= 1 && begin + count <= ((size_t)1 << k), "srs: shard [begin, begin+count) outside the 2^k bases");
    H2B_REQUIRE(d_g || d_gl, "srs: both base arrays are null");
    h2b_srs* s = new h2b_srs();
    s->k = k;
    s->begin = begin;
    s->count = count;
    s->c = msm_choose_c_fixed(count);
    s->W = (255 + s->c - 1) / s->c;
    try {
        const void* src[2] = {d_g, d_gl};
        for (int b = 0; b < 2; b++) {
            if (!src[b]) continue;
            H2B_CUDA(cudaMalloc(&s->table[b], (size_t)s->W * count * 64));
            msm_build_table(ctx, src[b], count, s->c, s->W, s->table[b]);
        }
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) {
        srs_free(ctx, s);
        throw;
    }
    *out = s;
}
// rows [begin, begin + count) of the host bases g / g_lagrange (either may be null) staged in WS_BASES / WS_MISC2, then built
static void srs_stage_build(h2b_ctx* ctx, const uint64_t* g, const uint64_t* g_lagrange, uint32_t k, size_t begin, size_t count,
                            h2b_srs** out) {
    const uint64_t* host[2] = {g, g_lagrange};
    const int slot[2] = {WS_BASES, WS_MISC2};
    const void* dev[2] = {nullptr, nullptr};
    for (int b = 0; b < 2; b++)
        if (host[b]) dev[b] = Staging(ctx, slot[b], count * 64).up(host[b] + 8 * begin, count * 64);
    srs_build(ctx, dev[0], dev[1], k, begin, count, out);
}

int h2b_srs_upload(h2b_ctx* ctx, const uint64_t* g, const uint64_t* g_lagrange, uint32_t k, size_t begin, size_t count,
                   h2b_srs** out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(k <= 27 && count >= 1 && begin + count <= ((size_t)1 << k), "srs: bad shard");
        if (ctx->members.size() <= 1) return srs_stage_build(ctx, g, g_lagrange, k, begin, count, out);
        // device group: contiguous index ranges, one per device
        H2B_REQUIRE(out, "srs: null output handle");
        const size_t G = ctx->members.size();
        H2B_REQUIRE(count >= G, "srs: fewer bases than devices");
        h2b_srs* top = new h2b_srs();
        top->k = k;
        top->begin = begin;
        top->count = count;
        try {
            group_each(ctx, [&](h2b_ctx* mb, size_t i) {
                const size_t lo = begin + count * i / G, hi = begin + count * (i + 1) / G;
                h2b_srs* part = nullptr;
                srs_stage_build(mb, g, g_lagrange, k, lo, hi - lo, &part);
                top->parts.push_back(part);
            });
        } catch (...) {
            srs_free(ctx, top);
            throw;
        }
        top->c = top->parts[0]->c;
        top->W = top->parts[0]->W;
        *out = top;
    });
}
int h2b_srs_upload_dev(h2b_ctx* ctx, const void* d_g, const void* d_g_lagrange, uint32_t k, size_t begin, size_t count,
                       h2b_srs** out) {
    return guarded(ctx, [&] { srs_build(ctx, d_g, d_g_lagrange, k, begin, count, out); });
}
int h2b_srs_info(const h2b_srs* srs, int* window_bits, int* windows) {
    if (!srs || !window_bits || !windows) return H2B_ERR_ARG;
    *window_bits = srs->c;
    *windows = srs->W;
    return H2B_OK;
}
void h2b_srs_destroy(h2b_ctx* ctx, h2b_srs* srs) {
    if (!srs) return;
    // the parts of a device group's handle are reachable only through that group's context
    if (!ctx || ctx->members.size() != srs->parts.size()) srs->parts.clear();
    if (!ctx) return srs_free(nullptr, srs);
    std::lock_guard<std::mutex> lock(ctx->mu);
    srs_free(ctx, srs);
}

// ------------------------------------------------------------------------------------------------ MSM
static const void* srs_table(const h2b_srs* srs, int basis, size_t n) {
    H2B_REQUIRE(srs, "msm: null SRS handle");
    H2B_REQUIRE(basis == H2B_BASIS_MONOMIAL || basis == H2B_BASIS_LAGRANGE, "msm: basis must be 0 (monomial) or 1 (lagrange)");
    H2B_REQUIRE(srs->table[basis], "msm: this basis was not uploaded");
    H2B_REQUIRE(n == srs->count, "msm: scalar count must equal the SRS shard size");
    return srs->table[basis];
}

int h2b_msm_g1_dev(h2b_ctx* ctx, const h2b_srs* srs, int basis, const void* d_scalars, size_t n, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_scalars && d_out, "msm: null pointer");
        const void* t = srs_table(srs, basis, n);
        msm_run(ctx, t, n, srs->c, srs->W, srs->W, d_scalars, d_out);
    });
}
int h2b_msm_g1_bases_dev(h2b_ctx* ctx, const void* d_bases, const void* d_scalars, size_t n, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_bases && d_scalars && d_out && n >= 1, "msm: null pointer or n == 0");
        msm_run_adhoc(ctx, d_bases, n, d_scalars, d_out);
    });
}
int h2b_msm_g1_batch_dev(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const void* const* d_scalars, size_t m, size_t n,
                         void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(basis && d_scalars && d_out, "msm: null pointer");
        std::vector<const void*> tables(m);
        for (size_t j = 0; j < m; j++) {
            H2B_REQUIRE(d_scalars[j], "msm: null scalar column");
            tables[j] = srs_table(srs, basis[j], n);
        }
        msm_run_batch(ctx, tables.data(), n, srs->c, srs->W, d_scalars, m, d_out);
    });
}
// Enqueue only: the m partial commitments of this context's shard end up in its WS_OUT buffer (returned), lanes joined
// onto the context's stream.  `row0`: first row of the shard inside the caller's columns.
static void* msm_batch_enqueue(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const uint64_t* const* scalars, size_t m, size_t n,
                               size_t row0) {
    // validate everything before any stream is forked (a throw after the fork would leave the lanes unjoined)
    std::vector<const void*> tables(m);
    for (size_t j = 0; j < m; j++) {
        H2B_REQUIRE(scalars[j], "msm: null scalar column");
        tables[j] = srs_table(srs, basis[j], n);
    }
    // the columns are cut into groups that share one sort / accumulate / reduce pipeline (msm_run_group); a group's columns
    // are staged side by side in the lane's buffer
    constexpr int NL = h2b_ctx::NLANES;
    const size_t gsz = msm_group_size(ctx, n, m, srs->W);
    const size_t ngroups = (m + gsz - 1) / gsz;
    const size_t gmax = (m + ngroups - 1) / ngroups;
    const int nl = (int)(ngroups < (size_t)NL ? ngroups : (size_t)NL);
    void* stage[NL];
    for (int l = 0; l < nl; l++) {
        ctx->cur_lane = l;
        stage[l] = ctx->get(WS_SCALARS, gmax * n * 32);
    }
    ctx->cur_lane = 0;
    void* d_out = ctx->get(WS_OUT, m * 96);
    cudaStream_t cs = ctx->copy_stream, ks = ctx->stream;
    H2B_CUDA(cudaEventRecord(ctx->fork_ev, ks));
    H2B_CUDA(cudaStreamWaitEvent(cs, ctx->fork_ev, 0));
    for (int l = 0; l < nl; l++) H2B_CUDA(cudaStreamWaitEvent(ctx->lane_stream[l], ctx->fork_ev, 0));
    struct Join {  // joins the lanes back onto the caller's stream on every exit path
        h2b_ctx* c; cudaStream_t ks; int nl;
        ~Join() {
            c->stream = ks;
            c->cur_lane = 0;
            c->in_lane = false;
            for (int l = 0; l < nl; l++) {
                cudaEventRecord(c->lane_done[l], c->lane_stream[l]);
                cudaStreamWaitEvent(ks, c->lane_done[l], 0);
            }
        }
    };
    Join join{ctx, ks, nl};
    size_t j = 0;
    for (size_t g = 0; g < ngroups; g++) {
        const size_t cnt = m / ngroups + (g < m % ngroups ? 1 : 0);
        const int l = (int)(g % nl);
        if (g >= (size_t)nl) H2B_CUDA(cudaStreamWaitEvent(cs, ctx->lane_consumed[l], 0));
        const void* d_cols[16];
        for (size_t t = 0; t < cnt; t++) {
            d_cols[t] = (char*)stage[l] + t * n * 32;
            H2B_CUDA(cudaMemcpyAsync((void*)d_cols[t], scalars[j + t] + 4 * row0, n * 32, cudaMemcpyHostToDevice, cs));
        }
        H2B_CUDA(cudaEventRecord(ctx->lane_ready[l], cs));
        H2B_CUDA(cudaStreamWaitEvent(ctx->lane_stream[l], ctx->lane_ready[l], 0));
        ctx->stream = ctx->lane_stream[l];
        ctx->cur_lane = l;
        ctx->in_lane = true;
        msm_run_group(ctx, tables.data() + j, n, srs->c, srs->W, srs->W, d_cols, cnt, (char*)d_out + 96 * j, ctx->lane_consumed[l]);
        ctx->in_lane = false;
        j += cnt;
    }
    return d_out;
}
// the fused all-reduce kernel combines at most 16 points per launch
static void allreduce_chunked(h2b_ctx* ctx, void* d_points, size_t m) {
    for (size_t lo = 0; lo < m; lo += 16) peer_allreduce(ctx, (char*)d_points + 96 * lo, m - lo < 16 ? m - lo : 16);
}
// host columns -> m commitments on the host.  Uploads run on the copy stream into per-lane staging buffers; lane l's MSM
// waits for its upload and releases the buffer as soon as the scatter pass has consumed it.  `reduce`: combine the
// partial sums of all connected GPUs with the fused NVLink all-reduce kernel before the one device-to-host copy.
// On a device group (h2b_ctx_create_multi) the SRS handle is sharded over the devices: every device commits its row range
// of every column, the partial sums meet in the same all-reduce kernel over in-process peer mappings.
static void msm_batch_host(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const uint64_t* const* scalars, size_t m, size_t n,
                           uint64_t* out_xyz, bool reduce) {
    H2B_REQUIRE(basis && scalars && out_xyz, "msm: null pointer");
    H2B_REQUIRE(srs, "msm: null SRS handle");
    if (m == 0) return;
    uint64_t* h_out = (uint64_t*)ctx->get_pinned(0, m * 96);
    if (!srs->parts.empty()) {
        H2B_REQUIRE(srs->parts.size() == ctx->members.size(), "msm: this SRS handle belongs to another device group");
        H2B_REQUIRE(n == srs->count, "msm: scalar count must equal the SRS size");
        std::vector<void*> d_outs(ctx->members.size());
        group_each(ctx, [&](h2b_ctx* mb, size_t g) {
            const h2b_srs* part = srs->parts[g];
            d_outs[g] = msm_batch_enqueue(mb, part, basis, scalars, m, part->count, part->begin - srs->begin);
        });
        group_each(ctx, [&](h2b_ctx* mb, size_t g) { allreduce_chunked(mb, d_outs[g], m); });
        H2B_CUDA(cudaMemcpyAsync(h_out, d_outs[0], m * 96, cudaMemcpyDeviceToHost, ctx->stream));
        group_each(ctx, [&](h2b_ctx* mb, size_t) { H2B_CUDA(cudaStreamSynchronize(mb->stream)); });
        memcpy(out_xyz, h_out, m * 96);
        return;
    }
    void* d_out = msm_batch_enqueue(ctx, srs, basis, scalars, m, n, 0);
    cudaStream_t ks = ctx->stream;
    if (reduce && peer_connected(ctx)) allreduce_chunked(ctx, d_out, m);
    H2B_CUDA(cudaMemcpyAsync(h_out, d_out, m * 96, cudaMemcpyDeviceToHost, ks));
    H2B_CUDA(cudaStreamSynchronize(ks));
    memcpy(out_xyz, h_out, m * 96);
}
int h2b_msm_g1_batch(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const uint64_t* const* scalars, size_t m, size_t n,
                     uint64_t* out_xyz) {
    return guarded(ctx, [&] { msm_batch_host(ctx, srs, basis, scalars, m, n, out_xyz, false); });
}
int h2b_msm_g1_batch_reduced(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const uint64_t* const* scalars, size_t m, size_t n,
                             uint64_t* out_xyz) {
    return guarded(ctx, [&] { msm_batch_host(ctx, srs, basis, scalars, m, n, out_xyz, true); });
}
int h2b_msm_g1(h2b_ctx* ctx, const h2b_srs* srs, int basis, const uint64_t* scalars, size_t n, uint64_t out_xyz[12]) {
    const uint64_t* cols[1] = {scalars};
    const int bases[1] = {basis};
    if (!scalars) return guarded(ctx, [&] { H2B_REQUIRE(false, "msm: null pointer"); });
    return h2b_msm_g1_batch(ctx, srs, bases, cols, 1, n, out_xyz);
}
int h2b_msm_g1_bases(h2b_ctx* ctx, const uint64_t* bases, const uint64_t* scalars, size_t n, uint64_t out_xyz[12]) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(bases && scalars && out_xyz && n >= 1, "msm: null pointer or n == 0");
        Staging sb(ctx, WS_BASES, n * 64), ss(ctx, WS_SCALARS, n * 32), so(ctx, WS_OUT, 96);
        void *d_b = sb.up(bases, n * 64), *d_s = ss.up(scalars, n * 32), *d_o = so.take(96);
        msm_run_adhoc(ctx, d_b, n, d_s, d_o);
        uint64_t* h_out = (uint64_t*)ctx->get_pinned(0, 96);
        H2B_CUDA(cudaMemcpyAsync(h_out, d_o, 96, cudaMemcpyDeviceToHost, ctx->stream));
        so.finish();
        memcpy(out_xyz, h_out, 96);
    });
}
int h2b_g1_sum_dev(h2b_ctx* ctx, const void* d_points_xyz, size_t m, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_points_xyz && d_out, "g1_sum: null pointer");
        g1_sum_run(ctx, d_points_xyz, m, d_out);
    });
}
int h2b_g1_sum(h2b_ctx* ctx, const uint64_t* points_xyz, size_t m, uint64_t out_xyz[12]) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(points_xyz && out_xyz, "g1_sum: null pointer");
        Staging st(ctx, WS_MISC, m * 96 + 96);
        void *d_p = st.up(points_xyz, m * 96), *d_o = st.take(96);
        g1_sum_run(ctx, d_p, m, d_o);
        uint64_t* h_out = (uint64_t*)ctx->get_pinned(0, 96);
        H2B_CUDA(cudaMemcpyAsync(h_out, d_o, 96, cudaMemcpyDeviceToHost, ctx->stream));
        st.finish();
        memcpy(out_xyz, h_out, 96);
    });
}
int h2b_g1_normalize(h2b_ctx* ctx, uint64_t* points_xyz, size_t m) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(points_xyz, "g1_normalize: null pointer");
        if (m == 0) return;
        Staging st(ctx, WS_MISC, m * 96);
        g1_normalize_run(ctx, st.inout(points_xyz, m * 96), m);
        st.finish();
    });
}
int h2b_g1_fixed_base_mul_dev(h2b_ctx* ctx, const uint64_t base_xy[8], const void* d_scalars, size_t n, void* d_out_xy) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(base_xy && d_scalars && d_out_xy, "fixed_base_mul: null pointer");
        g1_fixed_base_mul_run(ctx, base_xy, d_scalars, n, d_out_xy);
    });
}
int h2b_g1_fixed_base_mul(h2b_ctx* ctx, const uint64_t base_xy[8], const uint64_t* scalars, size_t n, uint64_t* out_xy) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(base_xy && scalars && out_xy, "fixed_base_mul: null pointer");
        if (n == 0) return;
        Staging ss(ctx, WS_SCALARS, n * 32), so(ctx, WS_BASES, n * 64);
        void *d_s = ss.up(scalars, n * 32), *d_o = so.out(out_xy, n * 64);
        g1_fixed_base_mul_run(ctx, base_xy, d_s, n, d_o);
        so.finish();
    });
}

// ------------------------------------------------------------------------------------------------ peer all-reduce
int h2b_peer_create(h2b_ctx* ctx, int rank, int nranks, uint8_t handle_out[64]) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(handle_out, "peer: null pointer");
        peer_create(ctx, rank, nranks, handle_out);
    });
}
int h2b_peer_connect(h2b_ctx* ctx, const uint8_t* handles) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(handles, "peer: null pointer");
        peer_connect(ctx, handles);
    });
}
int h2b_g1_allreduce_dev(h2b_ctx* ctx, void* d_points_xyz, size_t m) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_points_xyz, "peer: null pointer");
        peer_allreduce(ctx, d_points_xyz, m);
    });
}

// ------------------------------------------------------------------------------------------------ NTT
int h2b_domain_omega(uint32_t k, uint64_t omega_out[4]) {
    if (!omega_out || k > 28) return H2B_ERR_ARG;
    domain_omega(k, omega_out, false);
    return H2B_OK;
}
enum NttKind { NTT_PLAIN, NTT_LAGRANGE_TO_COEFF, NTT_COEFF_TO_LAGRANGE, NTT_EXTENDED_TO_COEFF, NTT_COEFF_TO_EXTENDED };
// ntt_run's root, scaling and coset mode for each kind; NTT_PLAIN takes the caller's root and scaling
struct NttArgs {
    uint64_t w[4];
    int scale, coset;
    NttArgs(NttKind kind, uint32_t log_n, const uint64_t* omega = nullptr, int plain_scale = 0) {
        if (kind == NTT_PLAIN) {
            memcpy(w, omega, 32);
            scale = plain_scale;
            coset = 0;
            return;
        }
        const bool inverse = kind == NTT_LAGRANGE_TO_COEFF || kind == NTT_EXTENDED_TO_COEFF;
        domain_omega(log_n, w, inverse);
        scale = inverse;
        coset = kind == NTT_EXTENDED_TO_COEFF ? 2 : kind == NTT_COEFF_TO_EXTENDED ? 1 : 0;
    }
};
static void ntt_inplace_dev(h2b_ctx* ctx, void* d_a, uint32_t log_n, NttKind kind, const uint64_t* omega = nullptr, int scale = 0) {
    H2B_REQUIRE(d_a, "ntt: null pointer");
    H2B_REQUIRE(log_n <= 28, "ntt: log_n exceeds the two-adicity of Fr (28)");
    if (kind == NTT_PLAIN) H2B_REQUIRE(omega, "ntt: null omega");
    const NttArgs t(kind, log_n, omega, scale);
    ntt_run(ctx, d_a, (size_t)1 << log_n, d_a, log_n, t.w, t.scale, t.coset);
}
static void ntt_inplace_host(h2b_ctx* ctx, uint64_t* a, uint32_t log_n, NttKind kind, const uint64_t* omega = nullptr, int scale = 0) {
    H2B_REQUIRE(a, "ntt: null pointer");
    H2B_REQUIRE(log_n <= 28, "ntt: log_n exceeds the two-adicity of Fr (28)");
    const size_t bytes = ((size_t)1 << log_n) * 32;
    Staging st(ctx, WS_NTT_A, bytes);
    ntt_inplace_dev(ctx, st.inout(a, bytes), log_n, kind, omega, scale);
    st.finish();
}
int h2b_ntt_fr(h2b_ctx* ctx, uint64_t* a, uint32_t log_n, const uint64_t omega[4], int scale_by_n_inv) {
    return guarded(ctx, [&] { ntt_inplace_host(ctx, a, log_n, NTT_PLAIN, omega, scale_by_n_inv); });
}
int h2b_ntt_fr_dev(h2b_ctx* ctx, void* d_a, uint32_t log_n, const uint64_t omega[4], int scale_by_n_inv) {
    return guarded(ctx, [&] { ntt_inplace_dev(ctx, d_a, log_n, NTT_PLAIN, omega, scale_by_n_inv); });
}
int h2b_lagrange_to_coeff(h2b_ctx* ctx, uint64_t* a, uint32_t k) { return guarded(ctx, [&] { ntt_inplace_host(ctx, a, k, NTT_LAGRANGE_TO_COEFF); }); }
int h2b_coeff_to_lagrange(h2b_ctx* ctx, uint64_t* a, uint32_t k) { return guarded(ctx, [&] { ntt_inplace_host(ctx, a, k, NTT_COEFF_TO_LAGRANGE); }); }
int h2b_lagrange_to_coeff_dev(h2b_ctx* ctx, void* d_a, uint32_t k) { return guarded(ctx, [&] { ntt_inplace_dev(ctx, d_a, k, NTT_LAGRANGE_TO_COEFF); }); }
int h2b_coeff_to_lagrange_dev(h2b_ctx* ctx, void* d_a, uint32_t k) { return guarded(ctx, [&] { ntt_inplace_dev(ctx, d_a, k, NTT_COEFF_TO_LAGRANGE); }); }
int h2b_extended_to_coeff(h2b_ctx* ctx, uint64_t* a, uint32_t ext_k) { return guarded(ctx, [&] { ntt_inplace_host(ctx, a, ext_k, NTT_EXTENDED_TO_COEFF); }); }
int h2b_extended_to_coeff_dev(h2b_ctx* ctx, void* d_a, uint32_t ext_k) { return guarded(ctx, [&] { ntt_inplace_dev(ctx, d_a, ext_k, NTT_EXTENDED_TO_COEFF); }); }

static void coeff_to_extended_dev(h2b_ctx* ctx, const void* d_coeffs, size_t n_coeffs, uint32_t ext_k, void* d_out) {
    const NttArgs t(NTT_COEFF_TO_EXTENDED, ext_k);
    ntt_run(ctx, d_coeffs, n_coeffs, d_out, ext_k, t.w, t.scale, t.coset);
}
int h2b_coeff_to_extended_dev(h2b_ctx* ctx, const void* d_coeffs, size_t n_coeffs, uint32_t ext_k, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_coeffs && d_out, "coeff_to_extended: null pointer");
        H2B_REQUIRE(ext_k <= 28 && n_coeffs <= ((size_t)1 << ext_k), "coeff_to_extended: sizes out of range");
        coeff_to_extended_dev(ctx, d_coeffs, n_coeffs, ext_k, d_out);
    });
}
int h2b_coeff_to_extended(h2b_ctx* ctx, const uint64_t* coeffs, size_t n_coeffs, uint32_t ext_k, uint64_t* out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(coeffs && out, "coeff_to_extended: null pointer");
        H2B_REQUIRE(ext_k <= 28 && n_coeffs <= ((size_t)1 << ext_k), "coeff_to_extended: sizes out of range");
        const size_t bytes = ((size_t)1 << ext_k) * 32;
        Staging st(ctx, WS_NTT_A, bytes);
        void* d = st.up(coeffs, n_coeffs * 32, bytes);
        coeff_to_extended_dev(ctx, d, n_coeffs, ext_k, d);
        H2B_CUDA(cudaMemcpyAsync(out, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        st.finish();
    });
}

static void check_columns(const void* const* a, const void* const* b, size_t m) {
    for (size_t i = 0; i < m; i++) H2B_REQUIRE(a[i] && b[i], "ntt batch: null column");
}
// m transforms of one kind, in[i] -> out[i]; n_coeffs: the input length of NTT_COEFF_TO_EXTENDED (the other kinds transform
// 2^log_n elements in place)
static void ntt_batch(h2b_ctx* ctx, NttKind kind, const uint64_t* const* in, uint64_t* const* out, size_t m, uint32_t log_n,
                      size_t n_coeffs = 0) {
    H2B_REQUIRE(in && out, "ntt batch: null pointer");
    H2B_REQUIRE(log_n <= 28 && n_coeffs <= ((size_t)1 << log_n), "ntt batch: sizes out of range");
    if (m == 0) return;
    check_columns((const void* const*)in, (const void* const*)out, m);
    const size_t n = (size_t)1 << log_n, bytes = n * 32, n_in = kind == NTT_COEFF_TO_EXTENDED ? n_coeffs : n;
    const NttArgs t(kind, log_n);
    ntt_deal(ctx, in, out, m, [&](h2b_ctx* c, const uint64_t* const* vi, uint64_t* const* vo, size_t mc) {
        if (mc == 0) return;
        const int slots[3] = {WS_NTT_A, WS_NTT_C, WS_NTT_D};
        void* buf[3];
        for (int b = 0; b < 3; b++) buf[b] = c->get(slots[b], bytes);
        (void)c->get(WS_NTT_B, bytes);  // scratch of ntt_run: allocate before anything is in flight
        ntt_pipeline(c, vi, mc, buf, n_in * 32, [&](size_t, int b) { ntt_run(c, buf[b], n_in, buf[b], log_n, t.w, t.scale, t.coset); },
                     [&](size_t i, int b, cudaStream_t down) {
                         H2B_CUDA(cudaStreamWaitEvent(down, c->pipe_ev[b][1], 0));
                         H2B_CUDA(cudaMemcpyAsync(vo[i], buf[b], bytes, cudaMemcpyDeviceToHost, down));
                     });
    });
}
// lagrange_to_coeff followed by coeff_to_extended for m columns, fused: the coefficients go up once, stay on the device
// for the coset transform, and both results come down on the second copy stream while the next column computes.
static void ntt_fused_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k, uint32_t ext_k, uint64_t* const* ext_out) {
    H2B_REQUIRE(a && ext_out, "ntt batch: null pointer");
    H2B_REQUIRE(k <= ext_k && ext_k <= 28, "ntt batch: sizes out of range");
    if (m == 0) return;
    check_columns((const void* const*)a, (const void* const*)ext_out, m);
    const size_t n = (size_t)1 << k, ne = (size_t)1 << ext_k;
    const NttArgs inv(NTT_LAGRANGE_TO_COEFF, k), ext(NTT_COEFF_TO_EXTENDED, ext_k);
    ntt_deal(ctx, a, ext_out, m, [&](h2b_ctx* c, uint64_t* const* va, uint64_t* const* ve, size_t mc) {
        if (mc == 0) return;
        const int small_slots[3] = {WS_NTT_E, WS_NTT_F, WS_NTT_G}, big_slots[3] = {WS_NTT_A, WS_NTT_C, WS_NTT_D};
        void *sm[3], *big[3];
        for (int b = 0; b < 3; b++) {
            sm[b] = c->get(small_slots[b], n * 32);
            big[b] = c->get(big_slots[b], ne * 32);
        }
        (void)c->get(WS_NTT_B, ne * 32);  // scratch of ntt_run: allocate before anything is in flight
        ntt_pipeline(c, va, mc, sm, n * 32,
                     [&](size_t, int b) {
                         ntt_run(c, sm[b], n, sm[b], k, inv.w, inv.scale, inv.coset);
                         H2B_CUDA(cudaEventRecord(c->ev[b], c->stream));  // coefficients ready
                         ntt_run(c, sm[b], n, big[b], ext_k, ext.w, ext.scale, ext.coset);
                     },
                     [&](size_t i, int b, cudaStream_t down) {
                         H2B_CUDA(cudaStreamWaitEvent(down, c->ev[b], 0));
                         H2B_CUDA(cudaMemcpyAsync(va[i], sm[b], n * 32, cudaMemcpyDeviceToHost, down));
                         H2B_CUDA(cudaStreamWaitEvent(down, c->pipe_ev[b][1], 0));
                         H2B_CUDA(cudaMemcpyAsync(ve[i], big[b], ne * 32, cudaMemcpyDeviceToHost, down));
                     });
    });
}
int h2b_lagrange_to_coeff_and_extended_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k, uint32_t ext_k,
                                             uint64_t* const* ext_out) {
    return guarded(ctx, [&] { ntt_fused_batch(ctx, a, m, k, ext_k, ext_out); });
}
int h2b_lagrange_to_coeff_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k) {
    return guarded(ctx, [&] { ntt_batch(ctx, NTT_LAGRANGE_TO_COEFF, a, a, m, k); });
}
int h2b_coeff_to_lagrange_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k) {
    return guarded(ctx, [&] { ntt_batch(ctx, NTT_COEFF_TO_LAGRANGE, a, a, m, k); });
}
int h2b_coeff_to_extended_batch(h2b_ctx* ctx, const uint64_t* const* coeffs, size_t m, size_t n_coeffs, uint32_t ext_k,
                                uint64_t* const* out) {
    return guarded(ctx, [&] { ntt_batch(ctx, NTT_COEFF_TO_EXTENDED, coeffs, out, m, ext_k, n_coeffs); });
}

// ------------------------------------------------------------------------------------------------ assignment
int h2b_assign_columns_dev(h2b_ctx* ctx, const void* d_vcol, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k,
                           size_t ncols, void* d_cols) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_vcol || N == 0) && (d_cols || ncols == 0) && (break_points || nbp == 0), "assign: null pointer");
        assign_columns_run(ctx, d_vcol, N, break_points, nbp, k, ncols, d_cols);
    });
}
int h2b_assign_columns(h2b_ctx* ctx, const uint64_t* vcol, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k,
                       size_t ncols, uint64_t* cols) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((vcol || N == 0) && (cols || ncols == 0) && (break_points || nbp == 0), "assign: null pointer");
        H2B_REQUIRE(k <= 28, "assign: k out of range");
        const size_t out_bytes = (ncols << k) * 32;
        Staging si(ctx, WS_ASSIGN_IN, N * 32), so(ctx, WS_ASSIGN_OUT, out_bytes);
        void *d_in = si.up(vcol, N * 32), *d_out = so.out(cols, out_bytes);
        assign_columns_run(ctx, d_in, N, break_points, nbp, k, ncols, d_out);
        so.finish();
    });
}
// `Assigned<Fr>` records in, columns out: flatten (Zero / Trivial / Rational with one batched inversion) + the gather
int h2b_assign_columns_assigned_dev(h2b_ctx* ctx, const void* d_cells, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k,
                                    size_t ncols, void* d_cols) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_cells || N == 0) && (d_cols || ncols == 0) && (break_points || nbp == 0), "assign: null pointer");
        void* d_vals = ctx->get(WS_ASSIGN_IN, N * 32 + 64);
        uint32_t* d_stats = (uint32_t*)((char*)d_vals + ((N * 32 + 31) & ~(size_t)31));
        assigned_flatten_run(ctx, d_cells, N, d_vals, d_stats, 1);
        assign_columns_run(ctx, d_vals, N, break_points, nbp, k, ncols, d_cols);
    });
}
int h2b_assign_columns_assigned(h2b_ctx* ctx, const uint64_t* cells, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k,
                                size_t ncols, uint64_t* cols) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((cells || N == 0) && (cols || ncols == 0) && (break_points || nbp == 0), "assign: null pointer");
        H2B_REQUIRE(k <= 28, "assign: k out of range");
        const size_t out_bytes = (ncols << k) * 32;
        Staging si(ctx, WS_ASSIGN_IN, N * 72 + N * 32 + 128), so(ctx, WS_ASSIGN_OUT, out_bytes);
        void* d_in = si.up(cells, N * 72);
        void* d_vals = si.take(N * 32 + 32);
        uint32_t* d_stats = (uint32_t*)si.take(8);
        void* d_out = so.out(cols, out_bytes);
        assigned_flatten_run(ctx, d_in, N, d_vals, d_stats, 0);
        uint32_t st[2] = {0, 0};
        if (N) {
            uint32_t* bounce = (uint32_t*)ctx->get_pinned(2, 4096);
            H2B_CUDA(cudaMemcpyAsync(bounce, d_stats, 8, cudaMemcpyDeviceToHost, ctx->stream));
            H2B_CUDA(cudaStreamSynchronize(ctx->stream));
            st[0] = bounce[0];
            st[1] = bounce[1];
        }
        H2B_REQUIRE(st[1] == 0, "assign: a cell record carries a tag other than 0 (Zero), 1 (Trivial), 2 (Rational)");
        if (st[0]) assigned_flatten_run(ctx, d_in, N, d_vals, d_stats, 1);  // Rational cells present: with the batched inversion
        assign_columns_run(ctx, d_vals, N, break_points, nbp, k, ncols, d_out);
        so.finish();
    });
}
int h2b_assign_lookups_dev(h2b_ctx* ctx, const void* d_vals, size_t N, uint32_t k, size_t L, void* d_cols) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_vals || N == 0) && (d_cols || L == 0), "assign: null pointer");
        assign_lookups_run(ctx, d_vals, N, k, L, d_cols);
    });
}
int h2b_assign_lookups(h2b_ctx* ctx, const uint64_t* vals, size_t N, uint32_t k, size_t L, uint64_t* cols) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((vals || N == 0) && (cols || L == 0), "assign: null pointer");
        H2B_REQUIRE(k <= 28, "assign: k out of range");
        const size_t out_bytes = (L << k) * 32;
        Staging si(ctx, WS_ASSIGN_IN, N * 32), so(ctx, WS_ASSIGN_OUT, out_bytes);
        void *d_in = si.up(vals, N * 32), *d_out = so.out(cols, out_bytes);
        assign_lookups_run(ctx, d_in, N, k, L, d_out);
        so.finish();
    });
}
int h2b_eval_rational_dev(h2b_ctx* ctx, const void* d_num, const void* d_den, size_t n, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_num && d_den && d_out) || n == 0, "eval_rational: null pointer");
        eval_rational_batched_run(ctx, d_num, d_den, n, d_out);
    });
}
int h2b_apply_rational_dev(h2b_ctx* ctx, void* d_values, size_t N, const void* d_index, void* d_den, size_t R, uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_status && (d_values || N == 0) && ((d_index && d_den) || R == 0), "apply_rational: null pointer");
        apply_rational_run(ctx, d_values, N, (const uint64_t*)d_index, d_den, R, d_status);
    });
}
int h2b_assign_lookups_indexed_dev(h2b_ctx* ctx, const void* d_values, size_t N, const void* d_index, size_t n_lookup, uint32_t k, size_t L,
                                   void* d_cols, uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_status && (d_values || N == 0) && (d_index || n_lookup == 0) && (d_cols || L == 0), "assign_lookups_indexed: null pointer");
        assign_lookups_indexed_run(ctx, d_values, N, (const uint64_t*)d_index, n_lookup, k, L, d_cols, d_status);
    });
}
int h2b_eval_rational(h2b_ctx* ctx, const uint64_t* num, const uint64_t* den, size_t n, uint64_t* out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((num && den && out) || n == 0, "eval_rational: null pointer");
        if (n == 0) return;
        Staging st(ctx, WS_ASSIGN_IN, 3 * n * 32);
        void *d_num = st.up(num, n * 32), *d_den = st.up(den, n * 32), *d_out = st.out(out, n * 32);
        eval_rational_batched_run(ctx, d_num, d_den, n, d_out);
        st.finish();
    });
}

// ------------------------------------------------------------------------------------------------ grand products
int h2b_batch_invert_fr_dev(h2b_ctx* ctx, void* d_a, size_t n) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_a || n == 0, "batch_invert: null pointer");
        batch_invert_run(ctx, d_a, n);
    });
}
int h2b_batch_invert_fr(h2b_ctx* ctx, uint64_t* a, size_t n) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(a || n == 0, "batch_invert: null pointer");
        if (n == 0) return;
        Staging st(ctx, WS_ASSIGN_IN, n * 32);
        batch_invert_run(ctx, st.inout(a, n * 32), n);
        st.finish();
    });
}
int h2b_grand_product_fr_dev(h2b_ctx* ctx, const void* d_f, const uint64_t start[4], size_t n, void* d_z) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(((d_f && d_z) || n == 0) && start, "grand_product: null pointer");
        grand_product_run(ctx, d_f, start, n, d_z);
    });
}
int h2b_grand_product_fr(h2b_ctx* ctx, const uint64_t* f, const uint64_t start[4], size_t n, uint64_t* z) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(((f && z) || n == 0) && start, "grand_product: null pointer");
        if (n == 0) return;
        Staging st(ctx, WS_ASSIGN_IN, 2 * n * 32);
        void *d_f = st.up(f, n * 32), *d_z = st.out(z, n * 32);
        grand_product_run(ctx, d_f, start, n, d_z);
        st.finish();
    });
}

int h2b_flex_gate_fold_dev(h2b_ctx* ctx, const void* d_q_ext, const void* d_a_ext, const uint64_t y[4], uint32_t k, uint32_t ext_k,
                           void* d_acc) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_q_ext && d_a_ext && y && d_acc, "flex_gate: null pointer");
        flex_gate_fold_run(ctx, d_q_ext, d_a_ext, y, k, ext_k, d_acc);
    });
}
int h2b_flex_gate_fold(h2b_ctx* ctx, const uint64_t* q_ext, const uint64_t* a_ext, const uint64_t y[4], uint32_t k, uint32_t ext_k,
                       uint64_t* acc) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(q_ext && a_ext && y && acc, "flex_gate: null pointer");
        H2B_REQUIRE(ext_k <= 28, "flex_gate: extended_k out of range");
        const size_t bytes = ((size_t)1 << ext_k) * 32;
        Staging st(ctx, WS_NTT_A, 3 * bytes);
        void *d_q = st.up(q_ext, bytes), *d_a = st.up(a_ext, bytes), *d_acc = st.inout(acc, bytes);
        flex_gate_fold_run(ctx, d_q, d_a, y, k, ext_k, d_acc);
        st.finish();
    });
}

// ------------------------------------------------------------------------------------------------ keygen-side SRS utilities
int h2b_g_to_lagrange_dev(h2b_ctx* ctx, const void* d_g, uint32_t k, void* d_g_lagrange) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_g && d_g_lagrange, "g_to_lagrange: null pointer");
        g_to_lagrange_run(ctx, d_g, k, d_g_lagrange);
    });
}
int h2b_g_to_lagrange(h2b_ctx* ctx, const uint64_t* g, uint32_t k, uint64_t* g_lagrange) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(g && g_lagrange, "g_to_lagrange: null pointer");
        H2B_REQUIRE(k <= 28, "g_to_lagrange: k out of range");
        const size_t bytes = ((size_t)1 << k) * 64;
        Staging st(ctx, WS_BASES, 2 * bytes);
        void *d_g = st.up(g, bytes), *d_gl = st.out(g_lagrange, bytes);
        g_to_lagrange_run(ctx, d_g, k, d_gl);
        st.finish();
    });
}
int h2b_srs_setup_dev(h2b_ctx* ctx, const uint64_t tau[4], const uint64_t base_xy[8], uint32_t k, void* d_g, void* d_g_lagrange) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(tau && base_xy, "srs_setup: null pointer");
        srs_setup_run(ctx, tau, base_xy, k, d_g, d_g_lagrange);
    });
}
int h2b_srs_setup(h2b_ctx* ctx, const uint64_t tau[4], const uint64_t base_xy[8], uint32_t k, uint64_t* g, uint64_t* g_lagrange) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(tau && base_xy, "srs_setup: null pointer");
        H2B_REQUIRE(k <= 28, "srs_setup: k out of range");
        const size_t bytes = ((size_t)1 << k) * 64;
        Staging st(ctx, WS_BASES, 2 * bytes);
        void *d_g = st.out(g, bytes), *d_gl = st.out(g_lagrange, bytes);
        srs_setup_run(ctx, tau, base_xy, k, g ? d_g : nullptr, g_lagrange ? d_gl : nullptr);
        st.finish();
    });
}
int h2b_g1_check_on_curve_dev(h2b_ctx* ctx, const void* d_points_xy, size_t n, size_t* off_curve) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_points_xy || n == 0) && off_curve, "check_on_curve: null pointer");
        *off_curve = g1_count_off_curve_run(ctx, d_points_xy, n);
    });
}
int h2b_g1_check_on_curve(h2b_ctx* ctx, const uint64_t* points_xy, size_t n, size_t* off_curve) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((points_xy || n == 0) && off_curve, "check_on_curve: null pointer");
        void* d = Staging(ctx, WS_BASES, n * 64).up(points_xy, n * 64);
        *off_curve = g1_count_off_curve_run(ctx, d, n);  // returns the count: synchronised
    });
}
int h2b_g1_decompress_dev(h2b_ctx* ctx, const void* d_bytes, size_t n, void* d_out_xy, size_t* invalid) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(((d_bytes && d_out_xy) || n == 0) && invalid, "g1_decompress: null pointer");
        *invalid = g1_decompress_run(ctx, d_bytes, n, d_out_xy);
    });
}
int h2b_g1_decompress(h2b_ctx* ctx, const uint8_t* bytes, size_t n, uint64_t* out_xy, size_t* invalid) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(((bytes && out_xy) || n == 0) && invalid, "g1_decompress: null pointer");
        *invalid = 0;
        if (n == 0) return;
        Staging st(ctx, WS_BASES, n * 96);
        void *d_in = st.up(bytes, n * 32), *d_out = st.out(out_xy, n * 64);
        *invalid = g1_decompress_run(ctx, d_in, n, d_out);
        st.finish();
    });
}
// a params image: k (u32 little-endian), g and g_lagrange (2^k G1 points each), g2 and s_g2, with points of `g1` / `g2` bytes
static int params_view(const uint8_t* bytes, size_t len, size_t g1, size_t g2, uint32_t* k, size_t* g_offset, size_t* g_lagrange_offset,
                       size_t* g2_offset, size_t* s_g2_offset) {
    if (!bytes || !k || len < 4) return H2B_ERR_ARG;
    const uint32_t kk = (uint32_t)bytes[0] | ((uint32_t)bytes[1] << 8) | ((uint32_t)bytes[2] << 16) | ((uint32_t)bytes[3] << 24);
    if (kk > 28) return H2B_ERR_ARG;
    const size_t n = (size_t)1 << kk;
    if (len < 4 + 2 * n * g1 + 2 * g2) return H2B_ERR_ARG;
    *k = kk;
    if (g_offset) *g_offset = 4;
    if (g_lagrange_offset) *g_lagrange_offset = 4 + n * g1;
    if (g2_offset) *g2_offset = 4 + 2 * n * g1;
    if (s_g2_offset) *s_g2_offset = 4 + 2 * n * g1 + g2;
    return H2B_OK;
}
int h2b_params_processed_view(const uint8_t* bytes, size_t len, uint32_t* k, size_t* g_offset, size_t* g_lagrange_offset,
                              size_t* g2_offset, size_t* s_g2_offset) {
    return params_view(bytes, len, 32, 64, k, g_offset, g_lagrange_offset, g2_offset, s_g2_offset);
}
// `ParamsKZG::read` of a SerdeFormat::Processed image, device side: decompress g and g_lagrange (every point is thereby
// on the curve), build the MSM tables.  H2B_ERR_ARG on a malformed image or an invalid point encoding.
int h2b_srs_read_processed(h2b_ctx* ctx, const uint8_t* bytes, size_t len, size_t begin, size_t count, h2b_srs** out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(bytes && out, "srs_read: null pointer");
        uint32_t k = 0;
        size_t og = 0, ol = 0;
        H2B_REQUIRE(h2b_params_processed_view(bytes, len, &k, &og, &ol, nullptr, nullptr) == H2B_OK, "srs_read: not a SerdeFormat::Processed params image");
        const size_t n = (size_t)1 << k;
        if (count == 0 && begin == 0) count = n;
        H2B_REQUIRE(count >= 1 && begin + count <= n, "srs_read: shard outside the 2^k bases");
        Staging st(ctx, WS_BASES, count * (64 + 128));
        void *c_g = st.up(bytes + og + 32 * begin, count * 32), *c_gl = st.up(bytes + ol + 32 * begin, count * 32);
        void *d_g = st.take(count * 64), *d_gl = st.take(count * 64);
        const size_t bad = g1_decompress_run(ctx, c_g, count, d_g) + g1_decompress_run(ctx, c_gl, count, d_gl);
        H2B_REQUIRE(bad == 0, "srs_read: the params image holds an invalid G1 encoding");
        srs_build(ctx, d_g, d_gl, k, begin, count, out);
    });
}
int h2b_params_raw_view(const uint8_t* bytes, size_t len, uint32_t* k, size_t* g_offset, size_t* g_lagrange_offset, size_t* g2_offset,
                        size_t* s_g2_offset) {
    return params_view(bytes, len, 64, 128, k, g_offset, g_lagrange_offset, g2_offset, s_g2_offset);
}
int h2b_g1_compress_dev(h2b_ctx* ctx, const void* d_xy, size_t n, void* d_bytes) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_xy && d_bytes) || n == 0, "g1_compress: null pointer");
        g1_compress_run(ctx, d_xy, n, d_bytes);
    });
}
int h2b_g1_compress(h2b_ctx* ctx, const uint64_t* xy, size_t n, uint8_t* bytes) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((xy && bytes) || n == 0, "g1_compress: null pointer");
        if (n == 0) return;
        Staging st(ctx, WS_BASES, n * 96);
        void *d_in = st.up(xy, n * 64), *d_out = st.out(bytes, n * 32);
        g1_compress_run(ctx, d_in, n, d_out);
        st.finish();
    });
}
// `ParamsKZG::write`: u32 LE k | g | g_lagrange | g2 | s_g2 with G1 points of `g1` bytes and the caller's `g2_bytes` bytes of
// G2 encodings.  A null `out` asks for the size (no device work); otherwise *len is the capacity on entry, the size on return.
static int params_write(h2b_ctx* ctx, uint32_t k, size_t g1, size_t g2_bytes, const void* d_g, const void* d_gl, const uint8_t* g2,
                        uint8_t* out, size_t* len, const std::function<void(size_t, uint8_t*)>& bases) {
    if (!len || k > 28) return H2B_ERR_ARG;
    const size_t n = (size_t)1 << k, need = 4 + 2 * n * g1 + g2_bytes;
    if (!out) {
        *len = need;
        return H2B_OK;
    }
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_g && d_gl && g2, "params_write: null pointer");
        H2B_REQUIRE(*len >= need, "params_write: the buffer is shorter than the image");
        for (int i = 0; i < 4; i++) out[i] = (uint8_t)(k >> (8 * i));
        bases(n, out + 4);
        std::memcpy(out + 4 + 2 * n * g1, g2, g2_bytes);
        *len = need;
    });
}
int h2b_params_write_processed(h2b_ctx* ctx, const void* d_g, const void* d_g_lagrange, uint32_t k, const uint8_t g2[128], uint8_t* out,
                               size_t* len) {
    return params_write(ctx, k, 32, 128, d_g, d_g_lagrange, g2, out, len, [&](size_t n, uint8_t* dst) {
        // both bases compressed into one staging buffer, one download
        Staging st(ctx, WS_BASES, 2 * n * 32);
        char* d = st.out(dst, 2 * n * 32);
        g1_compress_run(ctx, d_g, n, d);
        g1_compress_run(ctx, d_g_lagrange, n, d + n * 32);
        st.finish();
    });
}
int h2b_params_write_raw(h2b_ctx* ctx, const void* d_g, const void* d_g_lagrange, uint32_t k, const uint8_t g2[256], uint8_t* out, size_t* len) {
    return params_write(ctx, k, 64, 256, d_g, d_g_lagrange, g2, out, len, [&](size_t n, uint8_t* dst) {
        // the bases already are the RawBytes layout (Montgomery limbs)
        H2B_CUDA(cudaMemcpyAsync(dst, d_g, n * 64, cudaMemcpyDeviceToHost, ctx->stream));
        H2B_CUDA(cudaMemcpyAsync(dst + n * 64, d_g_lagrange, n * 64, cudaMemcpyDeviceToHost, ctx->stream));
        H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    });
}

// ------------------------------------------------------------------------------------------------ lookup permutation
int h2b_permute_expression_pair_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                    void* d_permuted_input, void* d_permuted_table) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_input && d_table && d_permuted_input && d_permuted_table, "permute_expression_pair: null pointer");
        H2B_REQUIRE(d_input != d_permuted_input && d_table != d_permuted_table && d_input != d_permuted_table && d_table != d_permuted_input,
                    "permute_expression_pair: outputs must not alias inputs");
        if (permute_expression_pair_run(ctx, d_input, d_table, k, blinding_factors, d_permuted_input, d_permuted_table))
            throw StatusError{H2B_ERR_UNSATISFIED, "permute_expression_pair: an input value is not in the table (ConstraintSystemFailure)"};
    });
}
int h2b_permute_expression_pair_async_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                          void* d_permuted_input, void* d_permuted_table, uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_input && d_table && d_permuted_input && d_permuted_table && d_status, "permute_expression_pair: null pointer");
        H2B_REQUIRE(d_input != d_permuted_input && d_table != d_permuted_table && d_input != d_permuted_table && d_table != d_permuted_input,
                    "permute_expression_pair: outputs must not alias inputs");
        const uint32_t* v = permute_expression_pair_enqueue(ctx, d_input, d_table, k, blinding_factors, d_permuted_input, d_permuted_table);
        H2B_CUDA(cudaMemcpyAsync(d_status, v, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    });
}
int h2b_permute_expression_pair(h2b_ctx* ctx, const uint64_t* input, const uint64_t* table, uint32_t k, uint32_t blinding_factors,
                                uint64_t* permuted_input, uint64_t* permuted_table) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(input && table && permuted_input && permuted_table, "permute_expression_pair: null pointer");
        H2B_REQUIRE(k <= 28 && (size_t)blinding_factors + 1 < ((size_t)1 << k), "permute_expression_pair: no usable rows");
        const size_t u = ((size_t)1 << k) - (blinding_factors + 1), bytes = u * 32;
        Staging st(ctx, WS_ASSIGN_IN, 4 * bytes);
        void *d_in = st.up(input, bytes), *d_tab = st.up(table, bytes), *d_pin = st.out(permuted_input, bytes),
             *d_ptab = st.out(permuted_table, bytes);
        if (permute_expression_pair_run(ctx, d_in, d_tab, k, blinding_factors, d_pin, d_ptab))
            throw StatusError{H2B_ERR_UNSATISFIED, "permute_expression_pair: an input value is not in the table (ConstraintSystemFailure)"};
        st.finish();
    });
}

// ------------------------------------------------------------------------------------------------ quotient (general)
namespace {
// a host column of the quotient entry points uploaded into its staging
void* put_column(Staging& st, const void* host, size_t bytes) {
    H2B_REQUIRE(host, "quotient: null column");
    return st.up(host, bytes);
}
struct StagedGraph {
    h2b_graph g;
    std::vector<const void*> fixed, advice, instance;
    StagedGraph(const h2b_graph* src, Staging& st, size_t bytes) : g(*src) {
        H2B_REQUIRE((src->fixed || !src->n_fixed) && (src->advice || !src->n_advice) && (src->instance || !src->n_instance), "graph: null table");
        for (size_t i = 0; i < src->n_fixed; i++) fixed.push_back(put_column(st, src->fixed[i], bytes));
        for (size_t i = 0; i < src->n_advice; i++) advice.push_back(put_column(st, src->advice[i], bytes));
        for (size_t i = 0; i < src->n_instance; i++) instance.push_back(put_column(st, src->instance[i], bytes));
        g.fixed = fixed.data();
        g.advice = advice.data();
        g.instance = instance.data();
    }
};
size_t graph_columns(const h2b_graph* g) {
    H2B_REQUIRE(g, "graph: null pointer");
    return g->n_fixed + g->n_advice + g->n_instance;
}
}  // namespace

int h2b_quotient_graph_dev(h2b_ctx* ctx, const h2b_graph* graph, uint32_t k, uint32_t ext_k, void* d_values) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(graph && d_values, "quotient_graph: null pointer");
        quotient_graph_run(ctx, graph, k, ext_k, d_values);
    });
}
int h2b_quotient_graph(h2b_ctx* ctx, const h2b_graph* graph, uint32_t k, uint32_t ext_k, uint64_t* values) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(graph && values, "quotient_graph: null pointer");
        H2B_REQUIRE(ext_k <= 28, "quotient: extended_k out of range");
        const size_t bytes = ((size_t)1 << ext_k) * 32;
        Staging st(ctx, WS_NTT_A, (graph_columns(graph) + 1) * bytes);
        StagedGraph sg(graph, st, bytes);
        quotient_graph_run(ctx, &sg.g, k, ext_k, st.inout(values, bytes));
        st.finish();
    });
}
int h2b_lookup_fold_dev(h2b_ctx* ctx, const h2b_graph* graph, const void* d_z, const void* d_permuted_input,
                        const void* d_permuted_table, const void* d_l0, const void* d_l_last, const void* d_l_active, uint32_t k,
                        uint32_t ext_k, void* d_values) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(graph && d_z && d_permuted_input && d_permuted_table && d_l0 && d_l_last && d_l_active && d_values, "lookup_fold: null pointer");
        lookup_fold_run(ctx, graph, d_z, d_permuted_input, d_permuted_table, d_l0, d_l_last, d_l_active, k, ext_k, d_values);
    });
}
int h2b_lookup_fold(h2b_ctx* ctx, const h2b_graph* graph, const uint64_t* z, const uint64_t* permuted_input,
                    const uint64_t* permuted_table, const uint64_t* l0, const uint64_t* l_last, const uint64_t* l_active, uint32_t k,
                    uint32_t ext_k, uint64_t* values) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(graph && values, "lookup_fold: null pointer");
        H2B_REQUIRE(ext_k <= 28, "quotient: extended_k out of range");
        const size_t bytes = ((size_t)1 << ext_k) * 32;
        Staging st(ctx, WS_NTT_A, (graph_columns(graph) + 7) * bytes);
        StagedGraph sg(graph, st, bytes);
        void* d[6];
        const void* host[6] = {z, permuted_input, permuted_table, l0, l_last, l_active};
        for (int i = 0; i < 6; i++) d[i] = put_column(st, host[i], bytes);
        lookup_fold_run(ctx, &sg.g, d[0], d[1], d[2], d[3], d[4], d[5], k, ext_k, st.inout(values, bytes));
        st.finish();
    });
}
int h2b_permutation_fold_dev(h2b_ctx* ctx, const void* const* d_z, size_t n_sets, const void* const* d_columns, const void* const* d_sigma,
                             size_t n_cols, size_t chunk_len, const void* d_l0, const void* d_l_last, const void* d_l_active,
                             const uint64_t beta[4], const uint64_t gamma[4], const uint64_t y[4], uint32_t blinding_factors, uint32_t k,
                             uint32_t ext_k, void* d_values) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(n_sets == 0 || (d_z && d_columns && d_sigma && d_l0 && d_l_last && d_l_active && d_values), "permutation_fold: null pointer");
        H2B_REQUIRE(beta && gamma && y, "permutation_fold: null challenge");
        permutation_fold_run(ctx, d_z, n_sets, d_columns, d_sigma, n_cols, chunk_len, d_l0, d_l_last, d_l_active, beta, gamma, y,
                             blinding_factors, k, ext_k, d_values);
    });
}
int h2b_permutation_fold(h2b_ctx* ctx, const uint64_t* const* z, size_t n_sets, const uint64_t* const* columns, const uint64_t* const* sigma,
                         size_t n_cols, size_t chunk_len, const uint64_t* l0, const uint64_t* l_last, const uint64_t* l_active,
                         const uint64_t beta[4], const uint64_t gamma[4], const uint64_t y[4], uint32_t blinding_factors, uint32_t k,
                         uint32_t ext_k, uint64_t* values) {
    return guarded(ctx, [&] {
        if (n_sets == 0) return;
        H2B_REQUIRE(z && columns && sigma && values && beta && gamma && y, "permutation_fold: null pointer");
        H2B_REQUIRE(ext_k <= 28, "quotient: extended_k out of range");
        const size_t bytes = ((size_t)1 << ext_k) * 32;
        Staging st(ctx, WS_NTT_A, (n_sets + 2 * n_cols + 4) * bytes);
        std::vector<const void*> dz, dc, ds;
        for (size_t i = 0; i < n_sets; i++) dz.push_back(put_column(st, z[i], bytes));
        for (size_t i = 0; i < n_cols; i++) dc.push_back(put_column(st, columns[i], bytes));
        for (size_t i = 0; i < n_cols; i++) ds.push_back(put_column(st, sigma[i], bytes));
        void *d0 = put_column(st, l0, bytes), *dl = put_column(st, l_last, bytes), *da = put_column(st, l_active, bytes),
             *dv = st.inout(values, bytes);
        permutation_fold_run(ctx, dz.data(), n_sets, dc.data(), ds.data(), n_cols, chunk_len, d0, dl, da, beta, gamma, y, blinding_factors,
                             k, ext_k, dv);
        st.finish();
    });
}

int h2b_divide_by_vanishing_poly_dev(h2b_ctx* ctx, void* d_values, uint32_t k, uint32_t ext_k) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_values, "divide_by_vanishing_poly: null pointer");
        divide_by_vanishing_run(ctx, d_values, k, ext_k);
    });
}
int h2b_divide_by_vanishing_poly(h2b_ctx* ctx, uint64_t* values, uint32_t k, uint32_t ext_k) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(values, "divide_by_vanishing_poly: null pointer");
        H2B_REQUIRE(ext_k <= 28, "quotient: extended_k out of range");
        const size_t bytes = ((size_t)1 << ext_k) * 32;
        Staging st(ctx, WS_NTT_A, bytes);
        divide_by_vanishing_run(ctx, st.inout(values, bytes), k, ext_k);
        st.finish();
    });
}

// ------------------------------------------------------------------------------------------------ constraint check
int h2b_check_graph_dev(h2b_ctx* ctx, const h2b_graph* g, uint32_t k, size_t rows, size_t max_report, void* d_report) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(g && d_report, "check_graph: null pointer");
        check_graph_run(ctx, g, k, rows, max_report, d_report);
    });
}
int h2b_check_lookup_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, size_t rows, size_t max_report,
                         void* d_report) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_input && d_table && d_report, "check_lookup: null pointer");
        check_lookup_run(ctx, d_input, d_table, k, rows, max_report, d_report);
    });
}
int h2b_permutation_decode_dev(h2b_ctx* ctx, const void* const* d_sigma, size_t n_cols, uint32_t k, void* d_map, size_t max_report,
                               void* d_reports) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_sigma && d_map && d_reports, "permutation_decode: null pointer");
        permutation_decode_run(ctx, d_sigma, n_cols, k, d_map, max_report, d_reports);
    });
}
int h2b_check_copies_dev(h2b_ctx* ctx, const void* const* d_columns, const void* d_map, size_t n_cols, uint32_t k, size_t max_report,
                         void* d_reports) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_columns && d_map && d_reports, "check_copies: null pointer");
        check_copies_run(ctx, d_columns, d_map, n_cols, k, max_report, d_reports);
    });
}

// ------------------------------------------------------------------------------------------------ MockProver of a builder
int h2b_mock_selectors_dev(h2b_ctx* ctx, const void* d_selectors, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t ncols,
                           void* d_q) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_selectors || N == 0) && (break_points || nbp == 0) && d_q, "mock_selectors: null pointer");
        mock_selectors_run(ctx, d_selectors, N, break_points, nbp, k, ncols, d_q);
    });
}
int h2b_mock_lookup_selector_dev(h2b_ctx* ctx, const void* d_index, size_t m, size_t N, size_t max_rows, uint32_t k, void* d_q,
                                 uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_index || m == 0) && d_q && d_status, "mock_lookup_selector: null pointer");
        mock_lookup_selector_run(ctx, (const uint64_t*)d_index, m, N, max_rows, k, d_q, d_status);
    });
}
int h2b_check_equalities_dev(h2b_ctx* ctx, const void* d_cells, size_t N, const void* d_pairs, size_t m, size_t max_report, void* d_report,
                             uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_cells || N == 0) && (d_pairs || m == 0) && d_report && d_status, "check_equalities: null pointer");
        check_equalities_run(ctx, d_cells, N, (const uint64_t*)d_pairs, m, max_report, d_report, d_status);
    });
}
int h2b_check_constants_dev(h2b_ctx* ctx, const void* d_cells, size_t N, const void* d_consts, const void* d_index, size_t m,
                            size_t max_report, void* d_report, uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_cells || N == 0) && ((d_consts && d_index) || m == 0) && d_report && d_status, "check_constants: null pointer");
        check_constants_run(ctx, d_cells, N, d_consts, (const uint64_t*)d_index, m, max_report, d_report, d_status);
    });
}
int h2b_count_distinct_dev(h2b_ctx* ctx, const void* d_values, size_t m, uint32_t* d_count) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_values || m == 0) && d_count, "count_distinct: null pointer");
        count_distinct_run(ctx, d_values, m, d_count);
    });
}

// ------------------------------------------------------------------------------------------------ keygen of a builder
int h2b_keygen_copies_nf_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                             const void* d_lookup_index, size_t n_lookup, const void* d_pairs, size_t M, const void* d_consts,
                             const void* d_const_index, size_t Mc, void* d_c, void* d_edges, uint32_t* d_status) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((break_points || nbp == 0) && (d_lookup_index || n_lookup == 0) && (d_pairs || M == 0) &&
                        ((d_consts && d_const_index) || Mc == 0) && (d_c || F == 0) && (d_edges || nbp + n_lookup + M + Mc == 0) && d_status,
                    "keygen_copies: null pointer");
        keygen_copies_run(ctx, N, break_points, nbp, k, F, A, L, (const uint64_t*)d_lookup_index, n_lookup, (const uint64_t*)d_pairs, M, d_consts,
                          (const uint64_t*)d_const_index, Mc, d_c, d_edges, d_status);
    });
}
int h2b_keygen_copies_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t A, size_t L,
                          const void* d_lookup_index, size_t n_lookup, const void* d_pairs, size_t M, const void* d_consts,
                          const void* d_const_index, size_t Mc, void* d_c, void* d_edges, uint32_t* d_status) {
    return h2b_keygen_copies_nf_dev(ctx, N, break_points, nbp, k, 1, A, L, d_lookup_index, n_lookup, d_pairs, M, d_consts, d_const_index, Mc, d_c,
                                    d_edges, d_status);
}
int h2b_keygen_instance_edges_nf_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                                     size_t usable, size_t I, const size_t* n_index, const void* d_index, void* d_edges, uint32_t* d_status) {
    return guarded(ctx, [&] {
        size_t total = 0;
        for (size_t m = 0; m < I && n_index; m++) total += n_index[m];
        H2B_REQUIRE((break_points || nbp == 0) && (n_index || I == 0) && (d_index || total == 0) && (d_edges || total == 0) &&
                        (d_status || I == 0),
                    "keygen_instance_edges: null pointer");
        keygen_instance_edges_run(ctx, N, break_points, nbp, k, F, A, L, usable, I, n_index, (const uint64_t*)d_index, d_edges, d_status);
    });
}
int h2b_keygen_instance_edges_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t A, size_t L,
                                  size_t usable, size_t I, const size_t* n_index, const void* d_index, void* d_edges, uint32_t* d_status) {
    return h2b_keygen_instance_edges_nf_dev(ctx, N, break_points, nbp, k, 1, A, L, usable, I, n_index, d_index, d_edges, d_status);
}
int h2b_keygen_sigma_map_dev(h2b_ctx* ctx, const void* d_edges, size_t E, size_t n_cols, uint32_t k, void* d_map) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_edges || E == 0) && d_map, "keygen_sigma_map: null pointer");
        keygen_sigma_map_run(ctx, d_edges, E, n_cols, k, d_map);
    });
}
int h2b_keygen_sigma_values_dev(h2b_ctx* ctx, const void* d_map, size_t n_cols, uint32_t k, void* d_sigma) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_map && d_sigma, "keygen_sigma_values: null pointer");
        keygen_sigma_values_run(ctx, d_map, n_cols, k, d_sigma);
    });
}

// ------------------------------------------------------------------------------------------------ opening arithmetic
// the value lands in WS_OUT and comes back to the host through pinned memory in both forms
static void eval_polynomial_to_host(h2b_ctx* ctx, const void* d_coeffs, size_t n, const uint64_t x[4], uint64_t out[4]) {
    void* d_out = ctx->get(WS_OUT, 32);
    eval_polynomial_run(ctx, d_coeffs, n, x, d_out);
    uint64_t* bounce = (uint64_t*)ctx->get_pinned(0, 4096);
    H2B_CUDA(cudaMemcpyAsync(bounce, d_out, 32, cudaMemcpyDeviceToHost, ctx->stream));
    H2B_CUDA(cudaStreamSynchronize(ctx->stream));
    memcpy(out, bounce, 32);
}
int h2b_eval_polynomial_dev(h2b_ctx* ctx, const void* d_coeffs, size_t n, const uint64_t x[4], uint64_t out[4]) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((d_coeffs || n == 0) && x && out, "eval_polynomial: null pointer");
        eval_polynomial_to_host(ctx, d_coeffs, n, x, out);
    });
}
int h2b_eval_polynomial(h2b_ctx* ctx, const uint64_t* coeffs, size_t n, const uint64_t x[4], uint64_t out[4]) {
    return guarded(ctx, [&] {
        H2B_REQUIRE((coeffs || n == 0) && x && out, "eval_polynomial: null pointer");
        eval_polynomial_to_host(ctx, Staging(ctx, WS_ASSIGN_IN, n * 32).up(coeffs, n * 32), n, x, out);
    });
}
int h2b_kate_division_dev(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t z[4], void* d_q) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_a && z && (d_q || n <= 1), "kate_division: null pointer");
        H2B_REQUIRE(d_a != d_q, "kate_division: q must not alias a");
        kate_division_run(ctx, d_a, n, z, d_q);
    });
}
int h2b_kate_division(h2b_ctx* ctx, const uint64_t* a, size_t n, const uint64_t z[4], uint64_t* q) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(a && z && (q || n <= 1), "kate_division: null pointer");
        H2B_REQUIRE(n >= 1, "kate_division: empty polynomial");  // before (n - 1) sizes the output
        if (n == 1) return;
        Staging st(ctx, WS_ASSIGN_IN, 2 * n * 32);
        void *d_a = st.up(a, n * 32), *d_q = st.out(q, (n - 1) * 32, n * 32);
        kate_division_run(ctx, d_a, n, z, d_q);
        st.finish();
    });
}
int h2b_kate_division_multi_dev(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t* points, size_t m, const uint64_t* weights,
                                void* d_q) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_a && points && weights && (d_q || n <= 1), "kate_division_multi: null pointer");
        H2B_REQUIRE(d_a != d_q, "kate_division_multi: q must not alias a");
        kate_division_multi_run(ctx, d_a, n, points, m, weights, d_q);
    });
}
int h2b_kate_division_multi(h2b_ctx* ctx, const uint64_t* a, size_t n, const uint64_t* points, size_t m, const uint64_t* weights,
                            uint64_t* q) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(a && points && weights && (q || n <= 1), "kate_division_multi: null pointer");
        H2B_REQUIRE(n >= 1, "kate_division_multi: empty polynomial");  // before (n - 1) sizes the output
        H2B_REQUIRE(m >= 1 && m <= H2B_KATE_MULTI_MAX, "kate_division_multi: 1..4 points");
        if (n == 1) return;
        Staging st(ctx, WS_ASSIGN_IN, 2 * n * 32);
        void *d_a = st.up(a, n * 32), *d_q = st.out(q, (n - 1) * 32, n * 32);
        kate_division_multi_run(ctx, d_a, n, points, m, weights, d_q);
        st.finish();
    });
}
int h2b_selector_conflicts_dev(h2b_ctx* ctx, const void* const* d_selectors, size_t S, uint32_t k, uint8_t* conflicts) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_selectors && conflicts, "selector_conflicts: null pointer");
        selector_conflicts_run(ctx, d_selectors, S, k, conflicts);
    });
}
int h2b_selector_conflicts(h2b_ctx* ctx, const uint64_t* const* selectors, size_t S, uint32_t k, uint8_t* conflicts) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(selectors && conflicts, "selector_conflicts: null pointer");
        H2B_REQUIRE(S >= 1 && S <= H2B_SELECTORS_MAX && k >= 1 && k <= 28, "selector_conflicts: 1..4096 columns, k in 1..28");
        const size_t bytes = ((size_t)32) << k;
        Staging st(ctx, WS_ASSIGN_IN, S * (bytes + 32));
        std::vector<const void*> d;
        for (size_t c = 0; c < S; c++) {
            H2B_REQUIRE(selectors[c], "selector_conflicts: null column");
            d.push_back(st.up(selectors[c], bytes));
        }
        selector_conflicts_run(ctx, d.data(), S, k, conflicts);
    });
}
int h2b_poly_lincomb_dev(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* scalars, size_t m, size_t n, void* d_out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(d_polys && scalars && (d_out || n == 0), "poly_lincomb: null pointer");
        poly_lincomb_run(ctx, d_polys, scalars, m, n, d_out);
    });
}
int h2b_poly_lincomb(h2b_ctx* ctx, const uint64_t* const* polys, const uint64_t* scalars, size_t m, size_t n, uint64_t* out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(polys && scalars && (out || n == 0), "poly_lincomb: null pointer");
        H2B_REQUIRE(m >= 1 && m <= 32, "poly_lincomb: 1..32 polynomials per call");
        if (n == 0) return;
        Staging st(ctx, WS_NTT_A, (m + 1) * n * 32);
        std::vector<const void*> dp;
        for (size_t j = 0; j < m; j++) dp.push_back(put_column(st, polys[j], n * 32));
        poly_lincomb_run(ctx, dp.data(), scalars, m, n, st.out(out, n * 32));
        st.finish();
    });
}

// ------------------------------------------------------------------------------------------------ test hook
int h2b_test_field_op(h2b_ctx* ctx, int field, int op, const uint64_t* a, const uint64_t* b, size_t n, uint64_t* out) {
    return guarded(ctx, [&] {
        H2B_REQUIRE(a && out && (b || (op > 2 && op < 7) || op == 9) && (field == 0 || field == 1) && op >= 0 && op <= 10, "field_op: bad argument");
        if (n == 0) return;
        const size_t in = (op == 10 ? 2 : 1) * n * 32;  // op 10 reads two operand pairs per output
        Staging st(ctx, WS_ASSIGN_IN, 2 * in + n * 32);
        void *d_a = st.up(a, in), *d_b = st.up(b, b ? in : 0, in), *d_out = st.out(out, n * 32);
        field_op_run(ctx, field, op, d_a, d_b, n, d_out);
        st.finish();
    });
}

}  // extern "C"
