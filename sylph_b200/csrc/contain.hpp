// contain.hpp — what the containment sources share (internal): the index (db_index.cu), the staged joins (contain.cu)
// and the query / profile calls (contain_calls.cu).
#pragma once

#include <functional>
#include <vector>

#include "common.cuh"

struct syl_db {
    int device = 0;
    syl_ctx *owner = nullptr;       // arrays are blocks of this ctx's cache
    cudaStream_t stream = nullptr;
    uint64_t n_genomes = 0;
    uint32_t genome_base = 0;
    uint64_t N = 0;             // index entries (genome_kmers + tracked)
    uint64_t *keys = nullptr;   // sorted ascending
    uint32_t *gid = nullptr;    // (genome << 1) | is_tracked
    uint32_t *bstart = nullptr; // NB + 1 bucket starts
    uint64_t NB = 0, M = 0, maxkey = 0;
    uint32_t *glen = nullptr;   // |genome_kmers| per genome (device)
    std::vector<uint64_t> h_gn_size;
    int has_tracked = 0;
    int k = 31;
    uint64_t c = 200;
};

namespace syl {

// bucket of the index directory that holds `key` (keys are uniform hashes: bucket = mulhi(key, M))
__device__ __forceinline__ uint64_t bucket_of(uint64_t key, uint64_t M, uint64_t NB) {
    uint64_t b = __umul64hi(key, M);
    return b < NB ? b : NB - 1;
}

// ---- the index (db_index.cu) ----------------------------------------------------------------

// The build's input: part 0 = genome k-mers, part 1 = tracked k-mers, each CSR over the same G genomes
// (off[part][0 .. G], validated: starts at 0, monotone).
struct DbInput {
    int mem;
    const uint64_t *keys[2], *off[2];
    uint64_t G, n[2];
};

int db_build(syl_ctx *ctx, const DbInput &in, const uint64_t *gn_size, int has_tracked, int k, uint64_t c, uint32_t genome_base,
             syl_db **out);
int check_db_size(uint64_t nk, uint64_t nt, uint64_t G);
int check_host_offsets(const uint64_t *kmer_off, const uint64_t *tracked_off, uint64_t G);

// ---- the joins (contain.cu) -----------------------------------------------------------------

struct SampleView {
    const uint64_t *hash;
    const uint32_t *count;
    uint64_t n;
};

// what -u needs to know about a sample (src/contain.rs:377-408)
struct SampleMeta { double mean_read_length; uint64_t c, sum_counts; };

constexpr uint32_t COV_BINS = 256;  // bins of the per-pair count histograms (histogram formulation)
constexpr int BOOT_ITERS = 100;

// Device bytes of one result row in the joins: two row tables, the bootstrap's results and its histogram
constexpr uint64_t ROW_BYTES = 2 * sizeof(syl_ani_row) + BOOT_ITERS * 17 + 17 * 4 + 8;

// What the joins of a host-sample batch may allocate beyond its plan (sample_batches.hpp charges neither): the CSR
// formulation's hit values (4 bytes per hit) and the row tables of a capacity retry.  The ctx's held plus transient
// device bytes stay within `limit` (0: unbounded, the handle path); a job that would pass it gives up with
// SPLIT_BATCH and contain_fast reruns its samples as two halves.  `want` is the refused allocation, `s0` the call's
// index of the job's first sample and `budget` the call's budget, for the error of a sample that does not fit alone.
struct JoinRoom {
    uint64_t limit = 0, budget = 0, want = 0;
    uint32_t s0 = 0;
};
constexpr int SPLIT_BATCH = -1;  // internal status, never returned through the C ABI

// The scan formulation of pass 1 (a query without an index): the genome k-mers of a chunk of whole genomes, on the
// device, probe every sample's lookup table (scan_plan.hpp has its layout).  The chunk's genomes are the db's of the
// call (n_genomes, genome_base, glen; it holds no index, N == 0); off = its n_genomes + 1 k-mer offsets, rebased to 0.
struct SampleTable {
    const uint64_t *hash;
    const uint32_t *count, *fp, *dir;
    uint64_t n, NB, M;
};
struct ScanChunk {
    const uint64_t *kmers, *off;
    uint64_t n;
    const SampleTable *tables;  // one per sample of the call
};

// the lookup tables of samples views[0 .. S) into tables (device, S entries), dir and fp (scan_plan.hpp), on the ctx
// stream; the host array `h` (S entries) is filled as well
int build_tables(syl_ctx *ctx, const SampleView *views, uint32_t S, DevBuf<SampleTable> &tables, DevBuf<uint32_t> &dir,
                 DevBuf<uint32_t> &fp, std::vector<SampleTable> &h);

// scan != nullptr: pass 1 of a query by the scan formulation (with profile: SYL_ERR_ARG)
int contain_fast(syl_ctx *ctx, const syl_db *db, const SampleView *views, const SampleMeta *metas, uint32_t n_samples,
                 const syl_contain_params *p, bool profile, std::vector<syl_ani_row> &out,
                 const std::function<int()> &overlap = {}, JoinRoom *room = nullptr, const ScanChunk *scan = nullptr);

// ---- the calls (contain_calls.cu) -----------------------------------------------------------

int check_contain_args(syl_ctx *ctx, int k, uint64_t c, bool has_tracked, bool profile, const syl_sample *const *samples,
                       uint32_t n_samples, const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);
int handle_views(syl_ctx *ctx, const syl_sample *const *samples, uint32_t n, bool unknown, std::vector<SampleView> &views,
                 std::vector<SampleMeta> &metas);
int copy_rows(const std::vector<syl_ani_row> &out, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);

}  // namespace syl
