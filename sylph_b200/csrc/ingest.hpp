// ingest.hpp — host-memory input to the device in bounded chunks, for read samples and genome batches alike.
//
// ASCII bases in (pinned or pageable) host memory are cut into chunks on record boundaries (the caller's plan); the
// ctx's worker pool packs chunk i+1.. into a ring of pinned staging buffers (exact BYTE_TO_SEQ codes, 16 bases per
// word; record offsets rebased to u32) while chunk i crosses PCIe and earlier chunks are seeded.  4.3 bytes of H2D
// traffic per 16 bases instead of 16.5 (SURVEY §8 f3).  Chunks may also cross the link as they are, through a two-slot
// device ring: every ASCII chunk when packing is off (SYL_HOST_INGEST=ascii), ASCII chunks taken from the back of the
// plan while the packers lag behind, and every chunk of caller 2-bit words.  A chunk marked `own` (a genome larger
// than a chunk) skips both rings: it is copied whole into a buffer of its own.
#pragma once

#include <functional>
#include <vector>

#include "common.cuh"

namespace syl {

// One mate's (or a single-end sample's, or a genome batch's) records: ASCII bytes or 2-bit words (nb bases either way),
// and the offsets of the records (off[i] - off_bias is the start of record i among the bases).  In host memory
// off_bias is 0; on the device it describes one seeding batch, whose off starts at the batch's first record.
struct Mate {
    const uint8_t *bases;
    const uint32_t *packed;
    uint64_t nb;
    const uint64_t *off;
    uint64_t off_bias;
};

constexpr int ING_SLOTS = 4;
constexpr uint64_t ING_CHUNK = 32ull << 20;        // bases per packed chunk (multiple of 16)
constexpr uint64_t ING_ASCII_CHUNK = 128ull << 20; // bases per chunk when every chunk is shipped as ASCII
constexpr uint64_t ING_MAXREC = 1ull << 19;        // records per packed chunk
// SYL_INGEST_CHUNK overrides the chunk size of either mode (tests; read per call)
uint64_t ingest_chunk(uint64_t dflt);
// Host ASCII: ship it as it is (true) or pack it on the host (SYL_HOST_INGEST; read per call)
bool host_ingest_ascii();

// Records (pairs) [r0, r1); per mate the first base and the number of bases.  A slot of either ring holds mate 1 at
// its start and mate 2 behind it at mate2_at(nb[0]) bases: one ring, one copy of the words and one of the offsets per
// chunk, whatever the number of mates.  Offsets: mate m's r1 - r0 + 1 entries start at entry m * (r1 - r0 + 1).
// own: the chunk goes through a device buffer of its own, with u64 offsets, instead of a ring slot (one mate only).
struct Chunk {
    uint64_t r0, r1, base[2], nb[2];
    bool own = false;
    uint64_t n_off() const { return r1 - r0 + 1; }
};

// records [r0, r1) per chunk: at most max_bases bases (of all mates together) and max_recs records, at least one record
void plan_chunks(const Mate *m, int n_mates, uint64_t n_reads, uint64_t max_bases, uint64_t max_recs,
                 std::vector<Chunk> &chunks);

// Receives chunk ci of the plan on the device: dm[i] holds mate i's bases (ASCII or 2-bit words), nb, u64 offsets and
// off_bias.  Chunks from the back of the plan may arrive before the ones in front of them.  The buffers stay valid
// until the work the sink enqueues on ctx->stream has run.
using ChunkSink = std::function<int(const Mate *dm, size_t ci)>;

// Host records m[0 .. n_mates) (ASCII, or 2-bit words in m[0].packed: one mate) -> chunks -> sink.  ascii_only: every
// ASCII chunk crosses the link as it is, front to back (1 byte of H2D traffic per base, no host packing).  2-bit words
// always do.  Else the pool packs the chunks.  Counts its H2D bytes and chunks into ctx->ingest_*.
int feed_host(syl_ctx *ctx, const Mate *m, int n_mates, const std::vector<Chunk> &chunks, bool ascii_only, const ChunkSink &sink);

// Device bytes of the staging rings once feed_host has grown them for this plan (allocated outside the block cache,
// kept until the ctx is destroyed; the ASCII ring of chunks taken from the back is counted whether or not it is used).
uint64_t ring_bytes_after(const syl_ctx *ctx, const std::vector<Chunk> &chunks, int n_mates, bool ascii_only);

// Host input staged into device slots while the ctx stream works on earlier ones (both rings above, host samples, scan
// and index-build chunks) crosses the link on the ctx's ONE copy stream, and a SlotHandoff hands each slot between the
// two streams.  ctx_copy_stream: *cs is that stream, created on first use with no ring; ingest_copy_stream: the same
// once the pinned ring exists.  ingest_copy copies `bytes` from src to dst on it, straight from pinned memory, from
// pageable memory through the pinned ring in slot-sized pieces (a pageable cudaMemcpyAsync would wait for the copy
// stream and block the calling thread).
int ctx_copy_stream(syl_ctx *ctx, cudaStream_t *cs);
int ingest_copy_stream(syl_ctx *ctx, cudaStream_t *cs);
int ingest_copy(syl_ctx *ctx, void *dst, const void *src, uint64_t bytes, bool pinned);

// The handoff of N device slots between the copy stream cs, which fills them, and the ctx stream st, which reads them.
// Per use of slot k: before_copy(k) (cs waits until st is done with k's last contents; a slot never used is free), the
// copies, copied_in(k) (on cs), take(k) (st waits for the copy; a slot may be staged well before it is taken), st's
// work on it, done(k) (on st).  fence(): cs waits once for st's work so far, for slots made of ctx-cache blocks.  The
// slots' buffers and which slot comes next stay with the user.  Declare it AFTER the slot buffers: its destructor
// drains cs, so the copies into cached blocks have run before those blocks go back to the ctx cache.
template <int N>
struct SlotHandoff {
    cudaStream_t cs = nullptr, st = nullptr;
    cudaEvent_t copied[N] = {}, used[N] = {};  // a host that waits on or polls the copy into slot k reads copied[k]
    SlotHandoff() = default;
    SlotHandoff(const SlotHandoff &) = delete;
    SlotHandoff &operator=(const SlotHandoff &) = delete;
    ~SlotHandoff() {
        if (cs) cudaStreamSynchronize(cs);
        for (int k = 0; k < N; k++)
            for (cudaEvent_t e : {copied[k], used[k]})
                if (e) cudaEventDestroy(e);
    }
    int init(cudaStream_t copy_stream, cudaStream_t ctx_stream) {
        cs = copy_stream;
        st = ctx_stream;
        for (int k = 0; k < N; k++) {
            SYL_CUDA(cudaEventCreateWithFlags(&copied[k], cudaEventDisableTiming));
            SYL_CUDA(cudaEventCreateWithFlags(&used[k], cudaEventDisableTiming));
        }
        return SYL_OK;
    }
    int fence() { SYL_CUDA(cudaEventRecord(used[0], st)); SYL_CUDA(cudaStreamWaitEvent(cs, used[0], 0)); return SYL_OK; }
    int before_copy(int k) { SYL_CUDA(cudaStreamWaitEvent(cs, used[k], 0)); return SYL_OK; }
    int copied_in(int k) { SYL_CUDA(cudaEventRecord(copied[k], cs)); return SYL_OK; }
    int take(int k) { SYL_CUDA(cudaStreamWaitEvent(st, copied[k], 0)); return SYL_OK; }
    int done(int k) { SYL_CUDA(cudaEventRecord(used[k], st)); return SYL_OK; }
};

}  // namespace syl
