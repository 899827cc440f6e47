// api.cu — the extern "C" boundary declared in include/sylph_b200.h (context + seeding entry
// points; the sketch / containment entry points live next to their kernels).
#include <algorithm>
#include <mutex>
#include <vector>
#include <new>

#include "common.cuh"
#include "host_pack.hpp"

namespace syl {

static thread_local std::string g_last_error;
thread_local syl_ctx *tl_ctx = nullptr;

static std::mutex g_live_mu;
static std::vector<syl_ctx *> g_live_ctx;  // contexts that still exist (handles may outlive their ctx)
static bool ctx_alive(syl_ctx *c) {
    std::lock_guard<std::mutex> lk(g_live_mu);
    return std::find(g_live_ctx.begin(), g_live_ctx.end(), c) != g_live_ctx.end();
}

int hblock_alloc(syl_ctx *ctx, void **p, size_t bytes) {
    bytes = (std::max<size_t>(bytes, 1) + 255) & ~(size_t)255;
    size_t best = (size_t)-1, bi = 0;
    for (size_t i = 0; i < ctx->free_blocks.size(); i++) {
        const size_t sz = ctx->free_blocks[i].second;
        if (sz >= bytes && sz < best) { best = sz; bi = i; }
    }
    if (best != (size_t)-1 && best <= 2 * bytes + (1u << 20)) {
        *p = ctx->free_blocks[bi].first;
        ctx->free_blocks[bi] = ctx->free_blocks.back();
        ctx->free_blocks.pop_back();
        ctx->handle_blocks[*p] = best;
        return SYL_OK;
    }
    cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) {
        *p = nullptr;
        set_error(std::string("cudaMalloc(") + std::to_string(bytes) + " B): " + cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? SYL_ERR_OOM : SYL_ERR_CUDA;
    }
    ctx->handle_blocks[*p] = bytes;
    ctx->cached_bytes += bytes;
    note_device_bytes(ctx);
    return SYL_OK;
}

void hblock_free(syl_ctx *ctx, void *p) {
    if (!p) return;
    if (ctx && ctx_alive(ctx)) {
        auto it = ctx->handle_blocks.find(p);
        if (it != ctx->handle_blocks.end()) {
            ctx->free_blocks.emplace_back(p, it->second);
            ctx->handle_blocks.erase(it);
            return;
        }
    }
    cudaFree(p);  // the owning ctx is gone (its cache was released without this block)
}
void set_error(const std::string &msg) { g_last_error = msg; }

int cache_trim(syl_ctx *ctx) {
    SYL_CUDA(cudaStreamSynchronize(ctx->stream));
    for (const auto &b : ctx->free_blocks) {
        cudaFree(b.first);
        ctx->cached_bytes -= b.second;
    }
    ctx->free_blocks.clear();
    return SYL_OK;
}

}  // namespace syl

using namespace syl;

extern "C" {

const char *syl_last_error(void) { return g_last_error.c_str(); }
int syl_abi_version(void) { return SYL_ABI_VERSION; }

int syl_ctx_create(int device, void *stream, syl_ctx **out) {
    if (!out) { set_error("out is NULL"); return SYL_ERR_ARG; }
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        set_error(std::string("no CUDA device: ") + cudaGetErrorString(e) + " (there is no CPU fallback)");
        return SYL_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) { set_error("bad device index"); return SYL_ERR_ARG; }
    SYL_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    SYL_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {  // sm_90a code runs on compute capability 9.0 only
        set_error(std::string("device ") + prop.name + " is sm_" + std::to_string(prop.major) +
                  std::to_string(prop.minor) + "; this library only carries sm_90a code");
        return SYL_ERR_CUDA;
    }
    syl_ctx *ctx = new (std::nothrow) syl_ctx();
    if (!ctx) return SYL_ERR_OOM;
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    if (stream) {
        ctx->stream = (cudaStream_t)stream;
        ctx->own_stream = false;
    } else {
        cudaError_t se = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        if (se != cudaSuccess) { delete ctx; set_error(cudaGetErrorString(se)); return SYL_ERR_CUDA; }
        ctx->own_stream = true;
    }
    // keep freed scratch in the pool instead of returning it to the driver on every sync
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t thresh = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh);
    }
    if (cudaMalloc((void **)&ctx->d_counters, CNT_SLOTS * sizeof(uint64_t)) != cudaSuccess ||
        cudaMallocHost((void **)&ctx->h_counters, CNT_SLOTS * sizeof(uint64_t)) != cudaSuccess) {
        set_error("ctx scratch allocation failed");
        syl_ctx_destroy(ctx);
        return SYL_ERR_OOM;
    }
    {
        std::lock_guard<std::mutex> lk(g_live_mu);
        g_live_ctx.push_back(ctx);
        note_context(+1);
    }
    *out = ctx;
    return SYL_OK;
}

void syl_ctx_destroy(syl_ctx *ctx) {
    if (!ctx) return;
    {
        std::lock_guard<std::mutex> lk(g_live_mu);
        const auto it = std::remove(g_live_ctx.begin(), g_live_ctx.end(), ctx);
        if (it != g_live_ctx.end()) note_context(-1);  // not when a failed syl_ctx_create cleans up
        g_live_ctx.erase(it, g_live_ctx.end());
    }
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    syl::ingest_destroy(ctx);
    for (auto &b : ctx->free_blocks) cudaFree(b.first);
    ctx->free_blocks.clear();
    if (syl::tl_ctx == ctx) syl::tl_ctx = nullptr;
    for (auto &t : ctx->timed_pending) { cudaEventDestroy(t.e0); cudaEventDestroy(t.e1); }
    for (auto e : ctx->event_pool) cudaEventDestroy(e);
    if (ctx->d_counters) cudaFree(ctx->d_counters);
    if (ctx->h_counters) cudaFreeHost(ctx->h_counters);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int syl_ctx_sync(syl_ctx *ctx) {
    if (!ctx) { set_error("ctx is NULL"); return SYL_ERR_ARG; }
    SYL_CUDA(cudaStreamSynchronize(ctx->stream));
    return SYL_OK;
}

uint64_t syl_ctx_launch_count(const syl_ctx *ctx) { return ctx ? ctx->launches : 0; }

int syl_ctx_device_bytes(syl_ctx *ctx, uint64_t *held, uint64_t *peak, int reset_peak) {
    if (!ctx) { set_error("ctx is NULL"); return SYL_ERR_ARG; }
    if (held) *held = ctx->cached_bytes;
    if (peak) *peak = ctx->peak_bytes;
    if (reset_peak) ctx->peak_bytes = ctx->cached_bytes + ctx->transient_bytes;
    return SYL_OK;
}

int syl_ctx_enable_timing(syl_ctx *ctx, int on) {
    if (!ctx) { set_error("ctx is NULL"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    ctx->timing = on != 0;
    return SYL_OK;
}

// resolve the recorded event pairs into the per-kernel totals (the stream must be idle)
static int timers_resolve(syl_ctx *ctx) {
    SYL_ENTER(ctx);
    if (ctx->timed_pending.empty()) return SYL_OK;
    SYL_CUDA(cudaStreamSynchronize(ctx->stream));
    for (auto &t : ctx->timed_pending) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess && t.which >= 0 && t.which < SYL_KERNEL_COUNT) {
            ctx->kernel_ms[t.which] += ms;
            ctx->kernel_launches[t.which]++;
        }
        ctx->event_pool.push_back(t.e0);
        ctx->event_pool.push_back(t.e1);
    }
    ctx->timed_pending.clear();
    return SYL_OK;
}

int syl_ctx_kernel_time(syl_ctx *ctx, int which, double *total_ms, uint64_t *launches, int reset) {
    if (!ctx || which < 0 || which >= SYL_KERNEL_COUNT) { set_error("bad argument"); return SYL_ERR_ARG; }
    SYL_TRY(timers_resolve(ctx));
    if (total_ms) *total_ms = ctx->kernel_ms[which];
    if (launches) *launches = ctx->kernel_launches[which];
    if (reset) { ctx->kernel_ms[which] = 0.; ctx->kernel_launches[which] = 0; }
    return SYL_OK;
}

int syl_ctx_seed_kernel_time(syl_ctx *ctx, double *total_ms, uint64_t *launches, uint64_t *bases, int reset) {
    if (!ctx) { set_error("ctx is NULL"); return SYL_ERR_ARG; }
    if (bases) *bases = ctx->seed_bases;
    if (reset) ctx->seed_bases = 0;
    return syl_ctx_kernel_time(ctx, SYL_KERNEL_SEED, total_ms, launches, reset);
}

static int seed_batch_impl(syl_ctx *ctx, int mem, const uint8_t *bases, const uint32_t *packed, uint64_t n_bases,
                           const uint64_t *rec_off, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos,
                           syl_survivor *out, uint64_t cap, uint64_t *n_out) {
    if (!ctx || !n_out || (!bases && !packed && n_bases) || !rec_off || (!out && cap)) {
        set_error("NULL argument");
        return SYL_ERR_ARG;
    }
    SYL_ENTER(ctx);
    *n_out = 0;
    cudaStream_t st = ctx->stream;
    Staged<uint8_t> sb;
    Staged<uint32_t> sp;
    Staged<uint64_t> so;
    if (packed) SYL_TRY(sp.init(ctx, mem, packed, (n_bases + 15) / 16));
    else SYL_TRY(sb.init(ctx, mem, bases, n_bases));
    SYL_TRY(so.init(ctx, mem, rec_off, n_rec + 1));
    DevBuf<syl_survivor> d_out;
    syl_survivor *dst = out;
    if (mem != SYL_MEM_DEVICE) {
        SYL_TRY(d_out.alloc(cap, st));
        dst = d_out.p;
    }
    SeedJob job;
    job.d_bases = packed ? nullptr : sb.p; job.d_packed = packed ? sp.p : nullptr; job.n_bases = n_bases;
    job.d_rec_off = so.p; job.off_bias = 0; job.n_rec = n_rec; job.k = k; job.c = c; job.sem = sem; job.with_pos = with_pos;
    job.d_out = dst; job.cap = cap;
    job.d_count = reinterpret_cast<unsigned long long *>(ctx->d_counters);
    SYL_CUDA(cudaMemsetAsync(ctx->d_counters, 0, 2 * sizeof(uint64_t), st));  // CNT_EVENTS, CNT_PENDING
    SYL_TRY(seed_enqueue(ctx, job));
    SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_EVENTS, ctx->d_counters + CNT_EVENTS, 8, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));
    *n_out = ctx->h_counters[CNT_EVENTS];
    if (*n_out > cap) { set_error("survivor buffer too small"); return SYL_ERR_CAPACITY; }
    if (mem != SYL_MEM_DEVICE && *n_out) {
        SYL_CUDA(cudaMemcpyAsync(out, d_out.p, *n_out * sizeof(syl_survivor), cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
    }
    return SYL_OK;
}

int syl_seed_batch(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                   const uint64_t *rec_off, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos,
                   syl_survivor *out, uint64_t cap, uint64_t *n_out) {
    return seed_batch_impl(ctx, mem, bases, nullptr, n_bases, rec_off, n_rec, k, c, sem, with_pos, out, cap, n_out);
}

int syl_seed_batch_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                           const uint64_t *rec_off, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos,
                           syl_survivor *out, uint64_t cap, uint64_t *n_out) {
    if (!packed && n_bases) { set_error("NULL argument"); return SYL_ERR_ARG; }
    return seed_batch_impl(ctx, mem, nullptr, packed, n_bases, rec_off, n_rec, k, c, sem, with_pos, out, cap, n_out);
}

}  // extern "C"
