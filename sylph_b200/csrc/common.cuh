// common.cuh — shared device/host helpers for the sylph_b200 kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/sylph_b200.h"

namespace syl {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const std::string &msg);

struct Status {
    int code;
    Status(int c = SYL_OK) : code(c) {}
    bool ok() const { return code == SYL_OK; }
};

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

// ---- context --------------------------------------------------------------------------------
}  // namespace syl

struct syl_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int num_sms = 132;
    uint64_t launches = 0;
    // small persistent scratch: device counters + pinned host mirror
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
    uint64_t ingest_h2d_bytes = 0, ingest_chunks_packed = 0, ingest_chunks_ascii = 0;  // last host-memory read sketch
    // HostIngest (sample.cu) of the host-memory read path: packer pool, copy stream, pinned ring of packed chunks
    // and two-slot device ring of ASCII chunks (lazily allocated, reused across calls)
    void *ingest = nullptr;
    // grow-only cache of scratch blocks: all work of a ctx is ordered on ONE stream, so a block can
    // be handed to the next user as soon as the previous user's kernels are enqueued; steady-state
    // calls then make no allocator calls at all (the CUDA allocators take driver-wide locks and
    // showed 30-500 ms stalls on shared hosts)
    std::vector<std::pair<void *, size_t>> free_blocks;
    std::unordered_map<void *, size_t> handle_blocks;  // blocks lent to sample / genomes / db handles
    size_t cached_bytes = 0;
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

// One survivor of a READ sketch as the dedup post-pass consumes it (32 bytes = one sector):
// recflag = read index << 1 | NO_PAIR, plus EV_PENDING while the pair keys still have to be
// computed from global memory (read not fully inside the seeding tile).
struct EventRec { uint64_t hash, recflag, p0, p1; };
static_assert(sizeof(EventRec) == 32, "EventRec is one 32-byte sector");
constexpr uint64_t NO_PAIR = 1ull;
constexpr uint64_t EV_PENDING = 1ull << 63;

constexpr uint32_t GRP_BPG = 32;  // hash buckets per read-sketch post-pass group (GroupOut in seed_kernel.cuh)

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
    uint32_t nbk = 0, ng = 0, slot = 0;
    unsigned long long *d_count = nullptr;  // running device counters: [0] survivors / events, [1] pending events
    // slotted survivor output (genome sketching): see SlotOut in seed_kernel.cuh
    uint32_t slot_cap = 0;
    uint32_t *d_tile_cnt = nullptr, *d_slot_overflow = nullptr;
};
uint64_t seed_cta_tiles(uint64_t n_bases);  // number of tiles of the seeding kernel
uint64_t seed_cta_tile_bases();             // window starts per tile of the seeding kernel
int seed_enqueue(syl_ctx *ctx, const SeedJob &job);
void ingest_destroy(syl_ctx *ctx);

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
        if (c) c->cached_bytes += bytes;
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
