// common.cuh — shared device/host helpers for the sylph_b200 kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <chrono>
#include <memory>
#include <new>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/sylph_b200.h"
#include "sample_parts.hpp"

namespace syl {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const std::string &msg);

#define SYL_CUDA(call)                                                                           \
    do {                                                                                         \
        cudaError_t _e = (call);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            ::syl::set_error(std::string(#call) + ": " + cudaGetErrorString(_e) + " (" +       \
                             __FILE__ + ":" + std::to_string(__LINE__) + ")");                   \
            return (_e == cudaErrorMemoryAllocation) ? SYL_ERR_OOM : SYL_ERR_CUDA;               \
        }                                                                                        \
    } while (0)

#define SYL_TRY(expr)                                                                            \
    do {                                                                                         \
        int _s = (expr);                                                                         \
        if (_s != SYL_OK) return _s;                                                             \
    } while (0)

// Entry of an API call on ctx: its device becomes current and DevBuf draws from its block cache.
#define SYL_ENTER(ctx)                                                                           \
    do {                                                                                         \
        SYL_CUDA(cudaSetDevice(ctx->device));                                                    \
        ::syl::tl_ctx = ctx;                                                                     \
    } while (0)

// ---- small host helpers -----------------------------------------------------------------------
inline unsigned nblk(uint64_t n, int bs) { return (unsigned)((n + bs - 1) / bs); }

// bits that hold every value up to maxval (at least 1)
inline int bits_for(uint64_t maxval) {
    int b = 1;
    while (b < 64 && (maxval >> b)) b++;
    return b;
}

// SYL_DEBUG_TIMING set: the host paths print where their time went (read once per process)
inline bool debug_timing() {
    static const bool on = getenv("SYL_DEBUG_TIMING") != nullptr;
    return on;
}
inline double ms_since(std::chrono::steady_clock::time_point t) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
}

// What a caller's pointer points into.  Memory CUDA does not know (the query fails; its error is cleared) is pageable.
enum class PtrKind { PAGEABLE, PINNED, DEVICE, MANAGED };
inline PtrKind ptr_kind(const void *p) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return PtrKind::PAGEABLE;
    }
    switch (at.type) {
        case cudaMemoryTypeHost: return PtrKind::PINNED;
        case cudaMemoryTypeDevice: return PtrKind::DEVICE;
        case cudaMemoryTypeManaged: return PtrKind::MANAGED;
        default: return PtrKind::PAGEABLE;
    }
}

// ---- context --------------------------------------------------------------------------------
}  // namespace syl

struct syl_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int num_sms = 132;
    uint64_t launches = 0;
    // small persistent scratch: device counters + pinned host mirror, slots named by syl::CounterSlot
    uint64_t *d_counters = nullptr;  // 32 x u64
    uint64_t *h_counters = nullptr;  // pinned
    // optional per-kernel timing (syl_ctx_enable_timing): every timed launch is bracketed by a pair of
    // CUDA events from a pool; the pairs are resolved (cudaEventElapsedTime) when the totals are read
    bool timing = false;
    struct TimedLaunch { int which; cudaEvent_t e0, e1; };
    std::vector<TimedLaunch> timed_pending;
    std::vector<cudaEvent_t> event_pool;
    double kernel_ms[SYL_KERNEL_COUNT] = {};
    uint64_t kernel_launches[SYL_KERNEL_COUNT] = {};
    uint64_t seed_bases = 0;
    uint64_t ingest_h2d_bytes = 0, ingest_chunks_packed = 0, ingest_chunks_ascii = 0;  // last host-memory sketch
    // HostIngest (ingest.cu): the copy stream of all host staging, and the host-memory read and genome paths' packer
    // pool, pinned ring of packed chunks and two-slot device ring of ASCII chunks (lazily allocated, reused across calls)
    void *ingest = nullptr;
    // grow-only cache of scratch blocks: all work of a ctx is ordered on ONE stream, so a block can
    // be handed to the next user as soon as the previous user's kernels are enqueued; steady-state
    // calls then make no allocator calls at all (the CUDA allocators take driver-wide locks and
    // showed 30-500 ms stalls on shared hosts)
    std::vector<std::pair<void *, size_t>> free_blocks;
    std::unordered_map<void *, size_t> handle_blocks;  // blocks lent to sample / genomes / db handles
    size_t cached_bytes = 0;     // every block the cache has allocated: free, lent to a handle or to a live DevBuf
    size_t transient_bytes = 0;  // live temporaries allocated outside the cache (the index build's)
    size_t peak_bytes = 0;       // high-water mark of cached_bytes + transient_bytes (syl_ctx_device_bytes)
    // read / pair sketches: device bytes a call may use (0: the free device memory at call time), and the number of
    // hash-range parts the last one was sketched in (sample_parts.hpp)
    uint64_t sample_budget = 0;
    uint32_t sample_parts = 0;
    uint64_t free_seen = 0;  // the device's free memory when a read sketch of this ctx last asked (cudaMemGetInfo)
};

namespace syl {
// RAII bracket of one timed launch (no-op unless syl_ctx_enable_timing is on)
struct KernelTimer {
    syl_ctx *c;
    int which;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    KernelTimer(syl_ctx *ctx, int w) : c(ctx), which(w) {
        if (!c->timing) return;
        auto take = [&]() {
            cudaEvent_t e = nullptr;
            if (!c->event_pool.empty()) { e = c->event_pool.back(); c->event_pool.pop_back(); }
            else if (cudaEventCreate(&e) != cudaSuccess) e = nullptr;
            return e;
        };
        e0 = take(); e1 = take();
        if (e0 && e1) cudaEventRecord(e0, c->stream);
    }
    void stop() {
        if (!e0 || !e1) return;
        cudaEventRecord(e1, c->stream);
        c->timed_pending.push_back({which, e0, e1});
        e0 = e1 = nullptr;
    }
    ~KernelTimer() { stop(); }
};
// ctx whose scratch cache DevBuf uses on this thread (set at every API entry)
extern thread_local syl_ctx *tl_ctx;
// device arrays owned by handles: taken from / returned to the owning ctx's block cache
int hblock_alloc(syl_ctx *ctx, void **p, size_t bytes);
void hblock_free(syl_ctx *ctx, void *p);
inline void note_device_bytes(syl_ctx *c) { c->peak_bytes = std::max(c->peak_bytes, c->cached_bytes + c->transient_bytes); }
}

// Device-resident SequencesSketch.kmer_counts (src/types.rs:145-155): parallel arrays sorted by hash
struct syl_sample {
    int device = 0;
    syl_ctx *owner = nullptr;       // arrays are blocks of this ctx's cache (free handles before their ctx)
    cudaStream_t stream = nullptr;
    uint64_t *hash = nullptr;  // ascending, distinct
    uint32_t *count = nullptr;
    uint64_t n = 0;
    int k = 31;
    uint64_t c = 200;
    double mean_read_length = 0.;
    uint64_t num_dup_removed = 0;
    uint64_t sum_counts = 0;   // sum of all counts (computed on first use: -u / estimate_covered_bases)
    bool sum_counts_valid = false;
};

// Device-resident batch of GenomeSketch (src/types.rs:163-173) in CSR form
struct syl_genomes {
    int device = 0;
    syl_ctx *owner = nullptr;       // arrays are blocks of this ctx's cache (free handles before their ctx)
    cudaStream_t stream = nullptr;
    uint64_t n = 0;                                       // genomes
    uint64_t *kmers = nullptr, *kmer_off = nullptr;       // genome_kmers, position order
    uint64_t *tracked = nullptr, *tracked_off = nullptr;  // pseudotax_tracked_nonused_kmers
    uint64_t *gn_size = nullptr;
    uint64_t total_kmers = 0, total_tracked = 0;
    int has_tracked = 0;
    int k = 31;
    uint64_t c = 200;
};

namespace syl {

// Slots of ctx->d_counters / h_counters, in slot order.  Two users of one slot never run within one call.
constexpr int CNT_SLOTS = 32;
enum CounterSlot : int {
    CNT_EVENTS = 0,          // seeding: survivors, or events in the overflow list (SeedJob::d_count[0])
    CNT_PENDING = 1,         // seeding: pending events (SeedJob::d_count[1]); the generic dedup's run count
    CNT_DUPS = 2,            // read sketch: duplicates removed
    CNT_PEND_MATE1 = 3,      // read sketch: CNT_PENDING before mate 1 of a batch
    CNT_UNIQ_TOTAL = 4,      // read sketch: in-kernel uniques (u64, summed by k_group_dedup)
    CNT_BACK_HALF = 4,       // genome back half: N, kept, tracked, slot overflow as four u32 over slots 4 and 5
    CNT_FALLBACK_TOTAL = 5,  // read sketch: slotted events of the fallback groups (u64, summed by k_group_dedup)
    CNT_KMER_TOTAL = 8,      // last k-mer offset of device CSR input
    CNT_TRACKED_TOTAL = 9,   // last tracked offset of device CSR input
    CNT_BAD_OFFSETS = 10,    // index build: device offsets that do not start at 0 or decrease
    CNT_COVS_TOTAL = 10,     // CSR formulation: coverage entries of pass 1
    CNT_MAX_KEY = 14,        // index build: largest key
    CNT_LARGE_BUCKETS = 15,  // index build: buckets of more than DB_MID entries
    CNT_PEND_MATE2 = 17,     // read sketch: CNT_PENDING before mate 2 of a batch
    CNT_SUM_COUNTS = 19,     // -u: sum of a sample's counts
};
static_assert(CNT_SUM_COUNTS < CNT_SLOTS, "the last slot is inside ctx->d_counters");
static_assert(CNT_DUPS == CNT_EVENTS + 2 && CNT_PEND_MATE1 == CNT_EVENTS + 3 && CNT_LARGE_BUCKETS == CNT_MAX_KEY + 1,
              "slots cleared or copied as one range");

// Owner of a half-built handle: frees it with the handle's free function unless release()d.  A half-built index is
// freed once the ctx stream has drained (db_index.cu).
struct HandleFree {
    void operator()(syl_sample *s) const { syl_sample_free(s); }
    void operator()(syl_genomes *g) const { syl_genomes_free(g); }
    void operator()(syl_db *db) const;
    void operator()(syl_profile_job *j) const { syl_profile_job_free(j); }
};
template <typename T>
using Handle = std::unique_ptr<T, HandleFree>;

// a new handle whose arrays will be blocks of ctx's cache, used on ctx's stream
template <typename T>
Handle<T> new_handle(syl_ctx *ctx) {
    Handle<T> h(new (std::nothrow) T());
    if (h) {
        h->device = ctx->device;
        h->owner = ctx;
        h->stream = ctx->stream;
    }
    return h;
}

// CSR k-mer arrays that their offsets count nk / nt entries in: one may be NULL only when it is empty (an empty torch
// tensor has no address)
inline int check_kmer_arrays(const uint64_t *kmers, uint64_t nk, const uint64_t *tracked, uint64_t nt) {
    if (nk && !kmers) { set_error("kmer_off counts k-mers but kmers is NULL"); return SYL_ERR_ARG; }
    if (nt && !tracked) { set_error("tracked_off counts tracked k-mers but tracked is NULL"); return SYL_ERR_ARG; }
    return SYL_OK;
}

// One survivor of a READ sketch as the dedup post-pass consumes it (32 bytes = one sector):
// recflag = read index << 1 | NO_PAIR, plus EV_PENDING while the pair keys still have to be
// computed from global memory (read not fully inside the seeding tile).
struct EventRec { uint64_t hash, recflag, p0, p1; };
static_assert(sizeof(EventRec) == 32, "EventRec is one 32-byte sector");
constexpr uint64_t NO_PAIR = 1ull;
constexpr uint64_t EV_PENDING = 1ull << 63;

// One batch for the seeding kernel (seed.cu: seed_enqueue).  Exactly one of d_bases (ASCII) / d_packed
// (2-bit words: base 16w+j of the batch in bits [30-2j, 31-2j] of word w) is set.
struct SeedJob {
    const uint8_t *d_bases = nullptr;
    const uint32_t *d_packed = nullptr;
    uint64_t n_bases = 0;
    const uint64_t *d_rec_off = nullptr;  // d_rec_off[i] - off_bias = start of record i inside the batch
    uint64_t off_bias = 0, n_rec = 0;
    int k = 31;
    uint64_t c = 200;
    int sem = SYL_SEM_AVX2, with_pos = 0;
    void *d_out = nullptr;                // syl_survivor[cap], or EventRec[ng * slot + cap] when emit_events
    uint64_t cap = 0;
    int emit_events = 0;
    uint64_t rec_base = 0;                // index of the batch's first read (events)
    int no_dedup = 0;
    uint32_t *d_pend = nullptr;           // indices of events whose pair keys are still missing
    uint32_t *d_group_cnt = nullptr;      // events: post-pass group counters (GroupOut in seed_kernel.cuh); nullptr = append
    uint64_t Mb = 0;
    uint32_t nbk = 0, ng = 0, slot = 0, g0 = 0;  // groups [g0, g0 + ng) of the map (Mb, nbk)
    uint64_t lo = 0, hi = ~0ull;                  // events: the hashes [lo, hi) (one part of the sample)
    unsigned long long *d_count = nullptr;  // running device counters: [0] survivors / events, [1] pending events
    // slotted survivor output (genome sketching): see SlotOut in seed_kernel.cuh
    uint32_t slot_cap = 0;
    uint32_t *d_tile_cnt = nullptr, *d_slot_overflow = nullptr;
};
uint64_t seed_cta_tiles(uint64_t n_bases);  // number of tiles of the seeding kernel
uint64_t seed_cta_tile_bases();             // window starts per tile of the seeding kernel
int seed_enqueue(syl_ctx *ctx, const SeedJob &job);
void ingest_destroy(syl_ctx *ctx);
// hand the ctx's cached free blocks back to the driver (waits for the ctx stream)
int cache_trim(syl_ctx *ctx);

// stream-ordered temporary device buffer (cudaMallocAsync from the device's default pool)
template <typename T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0, cap_bytes = 0;
    cudaStream_t s = nullptr;
    syl_ctx *owner = nullptr;  // ctx whose block cache the buffer came from (and goes back to)
    DevBuf() {}
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    int alloc(size_t count, cudaStream_t stream) {
        release();
        s = stream;
        n = count;
        size_t bytes = (std::max<size_t>(count, 1) * sizeof(T) + 255) & ~(size_t)255;
        syl_ctx *c = tl_ctx;
        owner = c;
        if (c) {  // best fit from the ctx cache
            size_t best = (size_t)-1, bi = 0;
            for (size_t i = 0; i < c->free_blocks.size(); i++) {
                const size_t sz = c->free_blocks[i].second;
                if (sz >= bytes && sz < best) { best = sz; bi = i; }
            }
            if (best != (size_t)-1 && best <= 2 * bytes + (1u << 20)) {
                p = reinterpret_cast<T *>(c->free_blocks[bi].first);
                cap_bytes = best;
                c->free_blocks[bi] = c->free_blocks.back();
                c->free_blocks.pop_back();
                return SYL_OK;
            }
        }
        cudaError_t e = cudaMalloc((void **)&p, bytes);
        if (e != cudaSuccess) {
            p = nullptr;
            set_error(std::string("cudaMalloc(") + std::to_string(bytes) + " B): " + cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? SYL_ERR_OOM : SYL_ERR_CUDA;
        }
        cap_bytes = bytes;
        if (c) {
            c->cached_bytes += bytes;
            note_device_bytes(c);
        }
        return SYL_OK;
    }
    void swap(DevBuf &o) {
        std::swap(p, o.p); std::swap(n, o.n); std::swap(cap_bytes, o.cap_bytes); std::swap(s, o.s); std::swap(owner, o.owner);
    }
    void release() {
        if (p) {
            if (owner) owner->free_blocks.emplace_back((void *)p, cap_bytes);  // not tl_ctx: two contexts on one thread never trade blocks
            else cudaFree(p);
        }
        p = nullptr;
        n = 0;
    }
};

// A whole caller input on the device: SYL_MEM_DEVICE pointers are used as they are, host memory is copied into a
// stream-ordered buffer with 64 bytes of padding past the end (the seeding kernel's bulk loads read past the last base).
template <typename T>
struct Staged {
    const T *p = nullptr;
    DevBuf<T> buf;
    int init(syl_ctx *ctx, int mem, const T *src, size_t n) {
        if (mem == SYL_MEM_DEVICE) { p = src; return SYL_OK; }
        if (mem != SYL_MEM_HOST) { set_error("bad mem"); return SYL_ERR_ARG; }
        SYL_TRY(buf.alloc(n + 64 / sizeof(T), ctx->stream));
        if (n) SYL_CUDA(cudaMemcpyAsync(buf.p, src, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        p = buf.p;
        return SYL_OK;
    }
};

// 16 two-bit fields (the even ones of 32, MSB-first) of x -> 32 bits
__device__ __forceinline__ uint32_t even_fields(uint64_t x) {
    x &= 0xCCCCCCCCCCCCCCCCull;
    x = (x | (x << 2)) & 0xF0F0F0F0F0F0F0F0ull;
    x = (x | (x << 4)) & 0xFF00FF00FF00FF00ull;
    x = (x | (x << 8)) & 0xFFFF0000FFFF0000ull;
    x = (x | (x << 16)) & 0xFFFFFFFF00000000ull;
    return (uint32_t)(x >> 32);
}

// ---- the reference's arithmetic, device side ------------------------------------------------

// src/types.rs:50-59 BYTE_TO_SEQ, as arithmetic (used off the hot path; the seeding kernel uses
// a shared-memory copy of the same 256-entry table, built from this function).
__host__ __device__ __forceinline__ uint32_t byte_to_seq(uint32_t b) {
    switch (b) {
        case 1: case 'C': case 'c': return 1u;
        case 2: case 'G': case 'g': return 2u;
        case 3: case 'T': case 't': case 'U': case 'u': return 3u;
        default: return 0u;
    }
}

// src/seeding.rs:4-15 — the shipped hash; line 7 negates the SUM key + (key << 21).
// Written with multiplies (k + (k<<21) == k * 0x200001 etc.) so that ptxas maps the four
// multiply steps to the FMA pipe (IMAD) and the three xor-shifts to the ALU pipe.
__host__ __device__ __forceinline__ uint64_t mm_hash64(uint64_t key) {
    key = ~(key * 0x200001ull);
    key ^= key >> 24;
    key *= 265ull;
    key ^= key >> 14;
    key *= 21ull;
    key ^= key >> 28;
    key *= 0x80000001ull;
    return key;
}

__host__ __device__ __forceinline__ uint64_t fmh_threshold(uint64_t c) {
    return 0xFFFFFFFFFFFFFFFFull / c;  // src/seeding.rs:108
}

// number of window START positions the reference visits in a record of length L
// (SURVEY §0 R2).  with_pos selects the positions-variant short-sequence rule.
__host__ __device__ __forceinline__ uint64_t valid_windows(uint64_t L, uint32_t k, int sem,
                                                           int with_pos) {
    if (L < k) return 0;
    if (sem == SYL_SEM_SCALAR) return L - k + 1;
    uint64_t min_len = with_pos ? 2ull * k : (uint64_t)k + 1;
    if (L < min_len) return 0;
    return 4ull * ((L - k + 1) / 4);
}

}  // namespace syl
