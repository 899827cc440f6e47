// host_pack.hpp — host side of the 2-bit ingest path (SURVEY §8 f3): exact BYTE_TO_SEQ packing of ASCII
// bases into the forward-stream words the seeding kernel consumes, spread over a persistent pool of
// worker threads that fills a ring of pinned staging buffers while earlier chunks cross PCIe.
#pragma once
#include <stdint.h>

#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

namespace syl {

// words[w] = sum_j BYTE_TO_SEQ[bases[16w + j]] << (30 - 2j)  (src/types.rs:50-59; bases past n read as 0)
// n_bases need not be a multiple of 16; ceil(n / 16) words are written.  Single thread.
void pack2_range(const uint8_t *bases, uint64_t n_bases, uint32_t *words);

// A unit of packing work: one slice of one chunk.
struct PackItem {
    const uint8_t *src;   // ASCII bases of the slice (slice starts at a multiple of 16 bases inside its chunk)
    uint64_t n;           // bases in the slice
    uint32_t *dst;        // destination words
    const uint64_t *off_src;  // or: a slice of record offsets to rebase into u32 (src == nullptr)
    uint64_t off_base, off_n;
    uint32_t *off_dst;
    uint32_t chunk;       // chunk the slice belongs to
};

// Persistent worker pool.  start() hands the items of a job (ordered by chunk) to the workers; an
// item of chunk c may only run once open_gate(g) with g >= c has been called (its pinned staging
// buffer is free again), and wait_chunk(c) returns when every item of chunk c is done, so that the
// caller can ship complete chunks while later ones are still being packed.  Workers and the caller
// BLOCK on condition variables while there is nothing to do (no spinning: on hosts with a CPU quota
// spinning threads burn the quota of the threads that have work).
class PackPool {
public:
    explicit PackPool(int n_threads);
    ~PackPool();
    int threads() const { return (int)workers_.size(); }
    // items / chunk_items stay owned by the caller and must outlive finish(); chunk_items[c] = items of chunk c
    void start(const std::vector<PackItem> *items, const std::vector<uint32_t> *chunk_items, int64_t gate);
    void open_gate(int64_t gate);
    void wait_chunk(uint32_t c);
    bool wait_chunk_for(uint32_t c, unsigned usec);  // true: chunk c is done; false: timed out
    bool chunk_done(uint32_t c);
    // take chunk c away from the workers if none of its items has been started; true: the caller handles it
    bool try_skip_chunk(uint32_t c);
    void finish();  // every item processed; must be called before the next start()

private:
    void worker();
    std::vector<std::thread> workers_;
    std::mutex mu_;
    std::condition_variable cv_work_, cv_done_;
    bool stop_ = false;
    const std::vector<PackItem> *items_ = nullptr;
    std::vector<uint32_t> remaining_;  // per chunk
    std::vector<uint32_t> taken_;      // per chunk: items handed out
    std::vector<uint8_t> skipped_;     // per chunk: taken over by the caller
    size_t next_ = 0, done_ = 0;
    int64_t gate_ = -1;
};

// Live contexts of this process (syl_ctx_create / syl_ctx_destroy): contexts share the host's cores and memory
// system, so the packer pool of a context and the ASCII-or-packed choice count them as well as LOCAL_WORLD_SIZE.
void note_context(int delta);
int live_contexts();  // at least 1

// Packer threads of a new pool: SYL_PACK_THREADS, else this process's share of the host (cores, container quota,
// LOCAL_WORLD_SIZE) divided by live_contexts().
int default_pack_threads();

}  // namespace syl
