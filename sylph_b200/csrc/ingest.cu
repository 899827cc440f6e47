// ingest.cu — the host-memory feeder of ingest.hpp: packer pool, copy stream, pinned ring of packed chunks, two-slot
// device ring of chunks shipped as they are, and the one-off buffer of a chunk larger than a ring slot.
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "host_pack.hpp"
#include "ingest.hpp"

namespace syl {

constexpr uint64_t ING_SLICE = 256ull << 10;       // bases per work item
constexpr uint64_t ING_OSLICE = 64ull << 10;       // offsets per work item

__global__ void k_off32_to_64(const uint32_t *__restrict__ in, uint64_t n, uint64_t *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
}

uint64_t ingest_chunk(uint64_t dflt) {
    if (const char *e = getenv("SYL_INGEST_CHUNK")) {
        const long long v = atoll(e);
        if (v >= 16) return (uint64_t)v & ~15ull;
    }
    return dflt;
}

// Packing costs host memory traffic (1.5 B per base: the packers read the ASCII, write the words, the copy engine reads
// them; ASCII costs 1 B per base), so it pays while PCIe is the narrow resource — 1 to 4 processes per host — and loses
// once the ranks of a host saturate its memory system instead (measured with 8 ranks on one host: 20.2 ms per 1 Gbp
// step shipping ASCII, 32.7 ms packing; with 1 and 2 ranks packing wins, 10.2 vs 19.9 and 16.4 vs 19.9 ms).
// The producers of a host are its processes (LOCAL_WORLD_SIZE) times the live contexts of each (several devices driven
// from one process).  SYL_HOST_INGEST = ascii | packed | packed-only overrides (read per call: the tests switch it at
// run time).
bool host_ingest_ascii() {
    const char *hi_env = getenv("SYL_HOST_INGEST");
    static const int local_ranks = []() { const char *e = getenv("LOCAL_WORLD_SIZE"); return e ? std::max(1, atoi(e)) : 1; }();
    return hi_env ? std::string(hi_env) == "ascii" : local_ranks * live_contexts() > 4;
}

// 256 bases: mate 2's words start 64-byte aligned and its ASCII 256-byte aligned (the seeding kernel's bulk copies need 16)
static uint64_t mate2_at(uint64_t nb1) { return (nb1 + 255) & ~255ull; }
static uint64_t footprint(const Chunk &c, int n_mates) { return n_mates == 2 ? mate2_at(c.nb[0]) + c.nb[1] : c.nb[0]; }
// caller 2-bit words of a chunk: from the word of its first base to the word of its last
static uint64_t word0(const Chunk &c) { return c.base[0] / 16; }
static uint64_t n_words(const Chunk &c) { return c.nb[0] ? (c.base[0] + c.nb[0] + 15) / 16 - word0(c) : 0; }
// bytes of a chunk shipped as it is
static uint64_t raw_bytes(const Chunk &c, int n_mates, bool words) { return words ? n_words(c) * 4 : footprint(c, n_mates); }

void plan_chunks(const Mate *m, int n_mates, uint64_t n_reads, uint64_t max_bases, uint64_t max_recs,
                 std::vector<Chunk> &chunks) {
    auto at = [&](uint64_t r) { return m[0].off[r] + (n_mates == 2 ? m[1].off[r] : 0); };
    uint64_t r0 = 0;
    while (r0 < n_reads) {
        const uint64_t base = at(r0);
        uint64_t lo = r0 + 1, hi = std::min(n_reads, r0 + max_recs);
        while (lo < hi) {
            const uint64_t mid = (lo + hi + 1) >> 1;
            if (at(mid) - base <= max_bases) lo = mid; else hi = mid - 1;
        }
        Chunk c{r0, lo, {0, 0}, {0, 0}};
        for (int i = 0; i < n_mates; i++) { c.base[i] = m[i].off[r0]; c.nb[i] = m[i].off[lo] - c.base[i]; }
        chunks.push_back(c);
        r0 = lo;
    }
}

struct HostIngest {
    // the ctx's copy stream (ingest.hpp); destroyed after the handoffs below have drained it
    std::unique_ptr<CUstream_st, cudaError_t (*)(cudaStream_t)> copy_stream{nullptr, cudaStreamDestroy};
    std::unique_ptr<PackPool> pool;
    // packed ring: words and chunk-relative u32 offsets, written by the pool
    uint32_t *h_words[ING_SLOTS] = {}, *h_off[ING_SLOTS] = {};  // pinned
    uint32_t *d_words[ING_SLOTS] = {}, *d_off32[ING_SLOTS] = {};
    uint64_t *d_off64[ING_SLOTS] = {};
    uint64_t cap_words = 0, cap_recs = 0;
    // ASCII ring: bases (or caller 2-bit words) and u64 offsets copied from caller memory as they are
    uint8_t *d_asc[2] = {};
    uint64_t *d_aoff[2] = {};
    uint64_t cap_asc = 0, cap_aoff = 0;
    int a_slot = 0, a_last = -1;  // next ASCII slot; slot of the latest ASCII copy (-1: none yet)
    int r_slot = 0;               // next packed-ring slot of ingest_copy's pageable pieces
    SlotHandoff<ING_SLOTS> packed;  // the packed ring's slots (also ingest_copy's pinned pieces)
    SlotHandoff<2> ascii;           // the ASCII ring's slots

    // the two streams that use the ring buffers: idle before a buffer is freed, and after a failed call
    void drain(cudaStream_t st) {
        cudaStreamSynchronize(st);
        cudaStreamSynchronize(copy_stream.get());
    }
    void free_packed() {
        for (int i = 0; i < ING_SLOTS; i++) {
            if (h_words[i]) cudaFreeHost(h_words[i]);
            if (h_off[i]) cudaFreeHost(h_off[i]);
            if (d_words[i]) cudaFree(d_words[i]);
            if (d_off32[i]) cudaFree(d_off32[i]);
            if (d_off64[i]) cudaFree(d_off64[i]);
            h_words[i] = h_off[i] = d_words[i] = d_off32[i] = nullptr;
            d_off64[i] = nullptr;
        }
        cap_words = cap_recs = 0;
    }
    void free_ascii() {
        for (int i = 0; i < 2; i++) {
            if (d_asc[i]) cudaFree(d_asc[i]);
            if (d_aoff[i]) cudaFree(d_aoff[i]);
            d_asc[i] = nullptr;
            d_aoff[i] = nullptr;
        }
        cap_asc = cap_aoff = 0;
    }
    // room for every chunk of the plan but the `own` ones, and for at least ING_CHUNK bases and 65536 records
    int ensure_packed(cudaStream_t st, const std::vector<Chunk> &chunks, int n_mates) {
        uint64_t words = ING_CHUNK / 16, recs = 65536;
        for (const Chunk &c : chunks) {
            if (c.own) continue;
            words = std::max(words, (footprint(c, n_mates) + 15) / 16);
            recs = std::max(recs, n_mates * c.n_off());
        }
        if (words <= cap_words && recs <= cap_recs) return SYL_OK;
        drain(st);
        const uint64_t w = std::max(words, cap_words), r = std::max(recs, cap_recs);
        free_packed();
        for (int i = 0; i < ING_SLOTS; i++) {
            SYL_CUDA(cudaMallocHost((void **)&h_words[i], (w + 16) * 4));
            SYL_CUDA(cudaMallocHost((void **)&h_off[i], (r + 16) * 4));
            SYL_CUDA(cudaMalloc((void **)&d_words[i], (w + 16) * 4));
            SYL_CUDA(cudaMalloc((void **)&d_off32[i], (r + 16) * 4));
            SYL_CUDA(cudaMalloc((void **)&d_off64[i], (r + 16) * 8));
        }
        cap_words = w;
        cap_recs = r;
        return SYL_OK;
    }
    // room for every chunk of the plan but the `own` ones (as ASCII, or as words), and for at least min_bytes bytes and
    // 65536 records
    int ensure_ascii(cudaStream_t st, const std::vector<Chunk> &chunks, int n_mates, bool words, uint64_t min_bytes) {
        uint64_t nb = min_bytes, recs = 65536;
        for (const Chunk &c : chunks) {
            if (c.own) continue;
            nb = std::max(nb, raw_bytes(c, n_mates, words));
            recs = std::max(recs, n_mates * c.n_off());
        }
        if (nb <= cap_asc && recs <= cap_aoff) return SYL_OK;
        drain(st);
        nb = std::max(nb, cap_asc);
        recs = std::max(recs, cap_aoff);
        free_ascii();
        for (int i = 0; i < 2; i++) {
            SYL_CUDA(cudaMalloc((void **)&d_asc[i], nb + 256));  // the seeding kernel's bulk loads read past the last base
            SYL_CUDA(cudaMalloc((void **)&d_aoff[i], (recs + 16) * 8));
        }
        cap_asc = nb;
        cap_aoff = recs;
        return SYL_OK;
    }
    // One chunk from caller memory through the ASCII ring and into the sink, as ASCII or as the caller's 2-bit words
    // (those start at the word of the chunk's first base: off_bias is that word's first base).  The copy of a slot
    // waits until the previous chunk in it is seeded; the record indices travel with the chunk, so chunks may go in
    // any order.
    int ship_ascii(syl_ctx *ctx, const Mate *m, int n_mates, const Chunk &c, size_t ci, const ChunkSink &sink) {
        const int slot = a_slot;
        a_slot ^= 1;
        const uint64_t no = c.n_off();
        const bool words = m[0].packed != nullptr;
        ascii.before_copy(slot);
        Mate bt[2] = {};
        for (int i = 0; i < n_mates; i++) {
            const void *src = words ? (const void *)(m[0].packed + word0(c)) : (const void *)(m[i].bases + c.base[i]);
            const uint64_t bytes = words ? n_words(c) * 4 : c.nb[i];
            uint8_t *dst = d_asc[slot] + (i ? mate2_at(c.nb[0]) : 0);
            if (words) bt[i] = {nullptr, reinterpret_cast<const uint32_t *>(dst), c.nb[i] + c.base[i] % 16, d_aoff[slot], word0(c) * 16};
            else bt[i] = {dst, nullptr, c.nb[i], d_aoff[slot] + i * no, c.base[i]};
            if ((bytes && cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, copy_stream.get()) != cudaSuccess) ||
                cudaMemcpyAsync((void *)bt[i].off, m[i].off + c.r0, no * 8, cudaMemcpyHostToDevice, copy_stream.get()) != cudaSuccess) {
                set_error("H2D copy failed");
                return SYL_ERR_CUDA;
            }
            ctx->ingest_h2d_bytes += bytes + no * 8;
        }
        if (words) ctx->ingest_chunks_packed++;
        else ctx->ingest_chunks_ascii++;
        ascii.copied_in(slot);
        ascii.take(slot);
        const int rc = sink(bt, ci);
        ascii.done(slot);
        a_last = slot;
        return rc;
    }
    ~HostIngest() {
        pool.reset();
        free_packed();
        free_ascii();
    }
};

void ingest_destroy(syl_ctx *ctx) {
    delete static_cast<HostIngest *>(ctx->ingest);
    ctx->ingest = nullptr;
}

// An `own` chunk (one mate): copied on the ctx stream into blocks of the ctx cache, as it is, with its u64 offsets.  It
// costs what staging the whole of it would, and leaves the rings at their size.
static int ship_own(syl_ctx *ctx, const Mate &m, const Chunk &c, size_t ci, const ChunkSink &sink) {
    cudaStream_t st = ctx->stream;
    const uint64_t no = c.n_off();
    DevBuf<uint8_t> b;
    DevBuf<uint32_t> w;
    DevBuf<uint64_t> off;
    SYL_TRY(off.alloc(no, st));
    SYL_CUDA(cudaMemcpyAsync(off.p, m.off + c.r0, no * 8, cudaMemcpyHostToDevice, st));
    Mate bt;
    uint64_t bytes = 0;
    if (m.packed) {
        bytes = n_words(c) * 4;
        SYL_TRY(w.alloc(n_words(c) + 16, st));
        if (bytes) SYL_CUDA(cudaMemcpyAsync(w.p, m.packed + word0(c), bytes, cudaMemcpyHostToDevice, st));
        bt = {nullptr, w.p, c.nb[0] + c.base[0] % 16, off.p, word0(c) * 16};
        ctx->ingest_chunks_packed++;
    } else {
        bytes = c.nb[0];
        SYL_TRY(b.alloc(c.nb[0] + 256, st));
        if (bytes) SYL_CUDA(cudaMemcpyAsync(b.p, m.bases + c.base[0], bytes, cudaMemcpyHostToDevice, st));
        bt = {b.p, nullptr, c.nb[0], off.p, c.base[0]};
        ctx->ingest_chunks_ascii++;
    }
    ctx->ingest_h2d_bytes += bytes + no * 8;
    return sink(&bt, ci);  // the buffers go back to the cache behind the sink's work on the same stream
}

int feed_host(syl_ctx *ctx, const Mate *m, int n_mates, const std::vector<Chunk> &chunks, bool ascii_only, const ChunkSink &sink) {
    cudaStream_t st = ctx->stream, cs = nullptr;
    SYL_TRY(ctx_copy_stream(ctx, &cs));
    HostIngest &I = *static_cast<HostIngest *>(ctx->ingest);
    const bool words = m[0].packed != nullptr;
    if (ascii_only || words) {
        SYL_TRY(I.ensure_ascii(st, chunks, n_mates, words, words ? ING_CHUNK / 4 : ING_ASCII_CHUNK));
        int rc = SYL_OK;
        for (size_t ci = 0; ci < chunks.size() && rc == SYL_OK; ci++)
            rc = chunks[ci].own ? ship_own(ctx, m[0], chunks[ci], ci, sink) : I.ship_ascii(ctx, m, n_mates, chunks[ci], ci, sink);
        if (rc != SYL_OK) I.drain(st);
        return rc;
    }
    for (const Chunk &c : chunks)  // the packed offsets are chunk-relative u32
        if (!c.own && (c.nb[0] >= 0xFFFFFFF0ull || c.nb[1] >= 0xFFFFFFF0ull)) { set_error("a single record of 4 GB or more"); return SYL_ERR_ARG; }
    // Two resources work in parallel: the packers (host memory bandwidth / CPU quota) and the PCIe link.  Packed
    // chunks are consumed from the front in order; whenever the front chunk is not packed yet and no ASCII copy
    // is in flight, a chunk nobody has started is taken from the BACK and shipped as ASCII (4x the bytes, but the
    // link would idle otherwise).  Needs pinned caller memory (a pageable copy would block this thread).
    bool steal_ok = true;
    for (int i = 0; i < n_mates; i++) steal_ok = steal_ok && ptr_kind(m[i].bases) == PtrKind::PINNED;
    {
        const char *e = getenv("SYL_HOST_INGEST");
        if (e && std::string(e) == "packed-only") steal_ok = false;
    }
    SYL_TRY(I.ensure_packed(st, chunks, n_mates));
    if (steal_ok) SYL_TRY(I.ensure_ascii(st, chunks, n_mates, false, ING_CHUNK));
    if (!I.pool) I.pool.reset(new PackPool(default_pack_threads()));
    std::vector<PackItem> items;
    std::vector<uint32_t> chunk_items(chunks.size());
    for (size_t ci = 0; ci < chunks.size(); ci++) {
        const Chunk &c = chunks[ci];
        const int slot = (int)(ci % ING_SLOTS);
        uint32_t n_items = 0;
        const uint64_t no = c.n_off();
        for (int i = 0; i < n_mates && !c.own; i++) {
            uint32_t *words = I.h_words[slot] + (i ? mate2_at(c.nb[0]) / 16 : 0);
            for (uint64_t o = 0; o < c.nb[i]; o += ING_SLICE, n_items++)
                items.push_back({m[i].bases + c.base[i] + o, std::min(ING_SLICE, c.nb[i] - o), words + o / 16, nullptr, 0, 0, nullptr, (uint32_t)ci});
            for (uint64_t o = 0; o < no; o += ING_OSLICE, n_items++)
                items.push_back({nullptr, 0, nullptr, m[i].off + c.r0 + o, c.base[i], std::min(ING_OSLICE, no - o), I.h_off[slot] + i * no + o, (uint32_t)ci});
        }
        chunk_items[ci] = n_items;
    }
    I.pool->start(&items, &chunk_items, ING_SLOTS - 1);
    const bool force_steal = getenv("SYL_INGEST_FORCE_STEAL") != nullptr;  // tests: alternate packed / ASCII chunks
    int rc = SYL_OK;
    int64_t f = 0, bk = (int64_t)chunks.size() - 1, last_packed = -1;
    bool steal_turn = true;  // force_steal only: alternate ASCII and packed chunks
    while (f <= bk && rc == SYL_OK) {
        if (chunks[(size_t)f].own) {  // ---- a chunk of its own (no pool items): in order, from the front
            rc = ship_own(ctx, m[0], chunks[(size_t)f], (size_t)f, sink);
            // every chunk up to f is done; the packed ones have crossed the link once the last of them has
            if (last_packed >= 0) cudaEventSynchronize(I.packed.copied[last_packed % ING_SLOTS]);
            I.pool->open_gate(f + ING_SLOTS);
            f++;
            continue;
        }
        const bool steal_first = force_steal && steal_ok && steal_turn;
        if (!steal_first && I.pool->chunk_done((uint32_t)f)) {  // ---- packed chunk from the front
            const size_t ci = (size_t)f;
            const Chunk &c = chunks[ci];
            const int slot = (int)(ci % ING_SLOTS);
            const uint64_t nw = (footprint(c, n_mates) + 15) / 16, no = n_mates * c.n_off();  // both mates in one copy each
            I.packed.before_copy(slot);  // the seeding of the previous chunk in this slot is done
            if (cudaMemcpyAsync(I.d_words[slot], I.h_words[slot], nw * 4, cudaMemcpyHostToDevice, cs) != cudaSuccess ||
                cudaMemcpyAsync(I.d_off32[slot], I.h_off[slot], no * 4, cudaMemcpyHostToDevice, cs) != cudaSuccess) {
                rc = SYL_ERR_CUDA; set_error("H2D copy failed"); break;
            }
            ctx->ingest_h2d_bytes += nw * 4 + no * 4;
            I.packed.copied_in(slot);
            I.packed.take(slot);
            k_off32_to_64<<<nblk(no, 256), 256, 0, st>>>(I.d_off32[slot], no, I.d_off64[slot]);
            ctx->launches++;
            Mate bt[2] = {};
            for (int i = 0; i < n_mates; i++)
                bt[i] = {nullptr, I.d_words[slot] + (i ? mate2_at(c.nb[0]) / 16 : 0), c.nb[i], I.d_off64[slot] + i * c.n_off(), 0};
            rc = sink(bt, ci);
            I.packed.done(slot);
            if (last_packed >= 0) {  // the pinned buffers of the previous packed chunk have crossed the link: refill them
                cudaEventSynchronize(I.packed.copied[last_packed % ING_SLOTS]);
                I.pool->open_gate(last_packed + ING_SLOTS);
            }
            last_packed = f;
            f++;
            ctx->ingest_chunks_packed++;
            steal_turn = true;
            continue;
        }
        const bool ascii_busy = !force_steal && I.a_last >= 0 && cudaEventQuery(I.ascii.copied[I.a_last]) == cudaErrorNotReady;
        if (steal_ok && !ascii_busy && (!force_steal || steal_turn) && bk > f && !chunks[(size_t)bk].own &&
            I.pool->try_skip_chunk((uint32_t)bk)) {  // ---- ASCII chunk from the back
            rc = I.ship_ascii(ctx, m, n_mates, chunks[(size_t)bk], (size_t)bk, sink);
            bk--;
            steal_turn = false;
            continue;
        }
        if (steal_first) { steal_turn = false; continue; }  // nothing to take from the back right now: go on with packed chunks
        // Front chunk still being packed.  If an ASCII copy is in flight and there are untouched chunks at the back,
        // whichever finishes first decides the next move (blocking on the packers alone would idle the link for as
        // long as they take: on a host whose memory system is shared by eight ranks that is most of the call).
        if (steal_ok && ascii_busy && bk > f) I.pool->wait_chunk_for((uint32_t)f, 40);
        else I.pool->wait_chunk((uint32_t)f);  // the packers are on it (or the only chunks left are theirs)
    }
    I.pool->open_gate((int64_t)1 << 60);  // all remaining items (skipped chunks included) drain
    I.pool->finish();
    if (debug_timing()) fprintf(stderr, "[host ingest] %zu chunks: %llu shipped as ASCII, %zu packed by %d threads\n", chunks.size(),
                     (unsigned long long)ctx->ingest_chunks_ascii, chunks.size() - (size_t)ctx->ingest_chunks_ascii, I.pool->threads());
    if (rc != SYL_OK) I.drain(st);
    return rc;
}

// the one place that creates the ctx's ingest state, its copy stream and the handoffs of both rings
int ctx_copy_stream(syl_ctx *ctx, cudaStream_t *cs) {
    if (!ctx->ingest) ctx->ingest = new HostIngest();
    HostIngest &I = *static_cast<HostIngest *>(ctx->ingest);
    if (!I.copy_stream) {
        SYL_CUDA(cudaStreamCreateWithFlags(cs, cudaStreamNonBlocking));
        I.copy_stream.reset(*cs);
        SYL_TRY(I.packed.init(*cs, ctx->stream));
        SYL_TRY(I.ascii.init(*cs, ctx->stream));
    }
    *cs = I.copy_stream.get();
    return SYL_OK;
}

int ingest_copy_stream(syl_ctx *ctx, cudaStream_t *cs) {
    SYL_TRY(ctx_copy_stream(ctx, cs));
    return static_cast<HostIngest *>(ctx->ingest)->ensure_packed(ctx->stream, {}, 1);
}

int ingest_copy(syl_ctx *ctx, void *dst, const void *src, uint64_t bytes, bool pinned) {
    HostIngest &I = *static_cast<HostIngest *>(ctx->ingest);
    ctx->ingest_h2d_bytes += bytes;
    if (pinned) {
        if (bytes) SYL_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, I.copy_stream.get()));
        return SYL_OK;
    }
    const uint64_t piece = I.cap_words * 4;
    for (uint64_t o = 0; o < bytes; o += piece) {
        const int slot = I.r_slot;
        I.r_slot = (I.r_slot + 1) % ING_SLOTS;
        const uint64_t n = std::min(piece, bytes - o);
        SYL_CUDA(cudaEventSynchronize(I.packed.copied[slot]));  // the slot's previous piece has crossed the link
        memcpy(I.h_words[slot], static_cast<const uint8_t *>(src) + o, n);
        SYL_CUDA(cudaMemcpyAsync(static_cast<uint8_t *>(dst) + o, I.h_words[slot], n, cudaMemcpyHostToDevice, I.copy_stream.get()));
        SYL_TRY(I.packed.copied_in(slot));
    }
    return SYL_OK;
}

uint64_t ring_bytes_after(const syl_ctx *ctx, const std::vector<Chunk> &chunks, int n_mates, bool ascii_only) {
    const HostIngest *I = static_cast<const HostIngest *>(ctx->ingest);
    uint64_t words = I ? I->cap_words : 0, recs = I ? I->cap_recs : 0, asc = I ? I->cap_asc : 0, aoff = I ? I->cap_aoff : 0;
    asc = std::max(asc, ascii_only ? ING_ASCII_CHUNK : ING_CHUNK);
    aoff = std::max<uint64_t>(aoff, 65536);
    if (!ascii_only) {
        words = std::max(words, ING_CHUNK / 16);
        recs = std::max<uint64_t>(recs, 65536);
    }
    for (const Chunk &c : chunks) {
        if (c.own) continue;
        asc = std::max(asc, footprint(c, n_mates));
        aoff = std::max(aoff, n_mates * c.n_off());
        if (ascii_only) continue;
        words = std::max(words, (footprint(c, n_mates) + 15) / 16);
        recs = std::max(recs, n_mates * c.n_off());
    }
    const uint64_t w = words ? (words + 16) * 4 : 0, r = recs ? recs + 16 : 0, a = asc + 256 + (aoff + 16) * 8;
    return ING_SLOTS * (w + r * 12) + 2 * a;
}

}  // namespace syl

using namespace syl;

extern "C" {

int syl_ctx_ingest_ring_bytes(const syl_ctx *ctx, uint64_t *device_bytes, uint64_t *pinned_bytes) {
    if (!ctx) { set_error("NULL argument"); return SYL_ERR_ARG; }
    const HostIngest *I = static_cast<const HostIngest *>(ctx->ingest);
    const uint64_t w = I && I->cap_words ? (I->cap_words + 16) * 4 : 0, r = I && I->cap_recs ? I->cap_recs + 16 : 0;
    const uint64_t a = I && I->cap_asc ? I->cap_asc + 256 + (I->cap_aoff + 16) * 8 : 0;
    if (device_bytes) *device_bytes = ING_SLOTS * (w + r * 12) + 2 * a;
    if (pinned_bytes) *pinned_bytes = ING_SLOTS * (w + r * 4);
    return SYL_OK;
}

int syl_ctx_ingest_stats(const syl_ctx *ctx, uint64_t *h2d_bytes, uint64_t *chunks_packed, uint64_t *chunks_ascii) {
    if (!ctx) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (h2d_bytes) *h2d_bytes = ctx->ingest_h2d_bytes;
    if (chunks_packed) *chunks_packed = ctx->ingest_chunks_packed;
    if (chunks_ascii) *chunks_ascii = ctx->ingest_chunks_ascii;
    return SYL_OK;
}

}  // extern "C"
