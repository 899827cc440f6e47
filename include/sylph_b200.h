/*
 * sylph_b200.h — C ABI of the H100-native (sm_90a) implementation of sylph's two hot paths:
 * FracMinHash sketching and containment query/profile.
 *
 * The reference (bluenote-1577/sylph v0.8.1, Rust) has no FFI or plugin interface; its backend
 * seam is the per-record runtime dispatch in src/sketch.rs:53-93 (AVX2 vs scalar) and the
 * per-pair call get_stats (src/contain.rs:601).  Per-record / per-pair granularity is far too
 * fine for a GPU, so this ABI sits one level up: one call per *batch* of records or pairs.
 * Each entry point names the reference function(s) it replaces.  A Rust maintainer binds these
 * with an `extern "C"` block (see INTEGRATION.md for the exact stub).
 *
 * Conventions
 *   - every function returns an int status (SYL_OK == 0); no exception/unwind crosses the ABI
 *     (reference convention: Option::None / log::error!+exit(1) / panic=abort, SURVEY §8-b);
 *     syl_last_error() gives a thread-local message for the last failure on this thread.
 *   - all sizes are uint64_t, all arrays little-endian POD, caller-allocated unless the name
 *     says otherwise.  `mem` tells where caller pointers live (SYL_MEM_HOST / SYL_MEM_DEVICE).
 *   - a syl_ctx owns one CUDA device + one stream; calls on one ctx are serialised by the
 *     caller (one ctx per rayon worker / per rank).  No global mutable state.
 *   - there is NO CPU fallback: if no compute capability 9.0 device / kernel image is available, calls
 *     fail with SYL_ERR_CUDA.
 *   - hard limits (reported as SYL_ERR_ARG, never silently wrapped): fewer than 2^32-2 records per batch,
 *     fewer than 2^32-2 survivor events per sample, fewer than 2^32-2 index entries (genome_kmers + tracked)
 *     and 2^31 genomes per db shard, fewer than 2^31 (sample, genome) pairs per syl_query / syl_profile call.
 *     Above 2^23 pairs per call the 256-bin per-pair histograms would exceed 8 GB: syl_query / syl_profile
 *     then run in the CSR formulation (slower, one more host synchronisation), the sharded profile (5)
 *     reports SYL_ERR_UNSUPPORTED.
 *   - handles (syl_sample / syl_genomes / syl_db / syl_profile_job) borrow device blocks from the ctx that
 *     created them: free them before their ctx, and use them with that ctx.
 */
#ifndef SYLPH_B200_H
#define SYLPH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SYL_ABI_VERSION 2

enum {
    SYL_OK = 0,
    SYL_ERR_ARG = 1,       /* bad argument (NULL, c == 0, offsets not monotone, ...) */
    SYL_ERR_CUDA = 2,      /* CUDA runtime / driver error, or no usable device */
    SYL_ERR_OOM = 3,       /* device or host allocation failed */
    SYL_ERR_CAPACITY = 4,  /* caller buffer too small; *n_out holds the needed size */
    SYL_ERR_UNSUPPORTED = 5 /* e.g. k not in {21,31} with AVX2 lane semantics: the reference
                               panics there (src/avx2_seeding.rs:46-52) */
};

enum { SYL_MEM_HOST = 0, SYL_MEM_DEVICE = 1 };

/* Which windows of a record are visited — the reference's two code paths:
 *   SYL_SEM_SCALAR  fmh_seeds: every one of the L-k+1 windows      (src/seeding.rs:86-146)
 *   SYL_SEM_AVX2    4 lanes of (L-k+1)/4 windows, the trailing (L-k+1)%4 windows dropped,
 *                   nothing for L < k+1 (hash-only) / L < 2k (positions)
 *                   (src/avx2_seeding.rs:33-44,152-162).  This is what sylph does on x86-64
 *                   and therefore the default everywhere in this library. */
enum { SYL_SEM_SCALAR = 0, SYL_SEM_AVX2 = 1 };

typedef struct syl_ctx syl_ctx;

const char *syl_last_error(void);
int syl_abi_version(void);

/* Create / destroy a context on CUDA device `device`.  `stream` may be NULL (the library
 * creates its own non-blocking stream) or an existing cudaStream_t passed as void* so a host
 * framework (e.g. torch) can order its own work with the library's. */
int syl_ctx_create(int device, void *stream, syl_ctx **out);
void syl_ctx_destroy(syl_ctx *ctx);
/* Block until everything queued on the ctx stream has finished. */
int syl_ctx_sync(syl_ctx *ctx);
/* Kernel launches issued by this ctx so far (bench.py's gpu_launches counter). */
uint64_t syl_ctx_launch_count(const syl_ctx *ctx);
/* Optional device-side timing of the dominant kernel (the seeding kernel): when enabled, every
 * launch is bracketed by CUDA events on the ctx stream; syl_ctx_seed_kernel_time returns the
 * accumulated milliseconds, launches and bases since the last reset (and resets when asked). */
int syl_ctx_enable_timing(syl_ctx *ctx, int on);
int syl_ctx_seed_kernel_time(syl_ctx *ctx, double *total_ms, uint64_t *launches, uint64_t *bases, int reset);
/* The same for the other kernels of the two paths (bench.py's live roofline figures): accumulated
 * CUDA-event milliseconds and launches of kernel class `which` since the last reset. Syncs the ctx stream. */
enum {
    SYL_KERNEL_SEED = 0,        /* k_seed (all variants) */
    SYL_KERNEL_GROUP_DEDUP = 1, /* read-sketch post-pass: k_group_dedup */
    SYL_KERNEL_JOIN = 2,        /* containment pass 1: k_join_hist (+ k_range_bounds, CSR formulation: k_join_csr) */
    SYL_KERNEL_JOIN2 = 3,       /* containment pass 2: k_join2_order (+ k_local_best when sharded) */
    SYL_KERNEL_STATS = 4,       /* k_stats_hist / k_stats */
    SYL_KERNEL_BOOT = 5,        /* bootstrap: k_boot_iter_p (+ k_boot_seq, k_boot_final) */
    SYL_KERNEL_GENOME_POST = 6, /* genome-sketch post-pass (everything after k_seed) */
    SYL_KERNEL_PACK = 7,        /* ASCII -> 2-bit packing on the device (unused by the host-packed path) */
    SYL_KERNEL_COUNT = 8
};
int syl_ctx_kernel_time(syl_ctx *ctx, int which, double *total_ms, uint64_t *launches, int reset);

/* ------------------------------------------------------------------------------------------
 * (1) Seeding — replaces extract_markers / extract_markers_positions over a whole batch
 *     (src/sketch.rs:53-93 -> src/avx2_seeding.rs:33-266, src/seeding.rs:86-209).
 *
 * bases   : n_bases ASCII bytes, all records concatenated (any case; every byte outside
 *           ACGTUacgtu and 0x01..0x03 reads as 'A', src/types.rs:50-59)
 * rec_off : n_rec+1 monotone offsets, rec_off[0] == 0, rec_off[n_rec] == n_bases
 * with_pos: 0 = extract_markers rule (nothing if L < k+1), 1 = extract_markers_positions rule
 *           (nothing if L < 2k).  Only matters for SYL_SEM_AVX2.
 * out     : survivors in unspecified order: hash, record index, index of the window's LAST
 *           base inside the record (what the reference's positions variant reports).
 *           Device-resident input pointers must be 16-byte aligned.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    uint64_t hash;
    uint32_t rec;
    uint32_t pos;
} syl_survivor;

int syl_seed_batch(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                   const uint64_t *rec_off, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos,
                   syl_survivor *out, uint64_t cap, uint64_t *n_out);

/* The same for 2-bit packed input (layout: see syl_sketch_reads_packed2). */
int syl_seed_batch_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                           const uint64_t *rec_off, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos,
                           syl_survivor *out, uint64_t cap, uint64_t *n_out);

/* ------------------------------------------------------------------------------------------
 * (2) Sample sketch — replaces sketch_sequences_needle's per-record loop
 *     (src/sketch.rs:917-947: pair_kmer_single :624-656, extract_markers,
 *     dup_removal_lsh_full_exact(.., Some(MAX_DEDUP_COUNT)) :690-731) for single-end reads
 *     already parsed into a flat buffer.  Result = the FxHashMap<Kmer,u32> of
 *     SequencesSketch (src/types.rs:145-155) as two parallel arrays sorted by hash,
 *     resident on the device.
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_sample syl_sample;

int syl_sketch_reads(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                     const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup,
                     int sem, syl_sample **out);
/* The same for reads that are already 2-bit packed: word w (little-endian u32) holds bases 16w .. 16w+15 of
 * the flat buffer, base 16w+j in bits [30-2j, 31-2j], codes = BYTE_TO_SEQ (src/types.rs:50-59: A/a 0, C/c 1,
 * G/g 2, T/t/U/u 3, everything else 0); ceil(n_bases/16) words; rec_off in bases as above.  A FASTQ parser
 * that packs while it parses ships 4x fewer bytes to the device.  syl_sketch_reads with SYL_MEM_HOST does
 * this internally (worker threads pack into pinned staging buffers while earlier chunks are copied and
 * seeded); SYL_PACK_THREADS overrides the worker count (default min(cores, 64)). */
int syl_sketch_reads_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                             const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup,
                             int sem, syl_sample **out);
/* Read pairs — replaces sketch_pair_sequences (src/sketch.rs:771-895) for `--fpr 0`, i.e. the EXACT
 * (k-mer, pair key) set with no count threshold (:829-838, :855-865): pair_kmer (:658-688) keys from the first 32
 * bases of both mates, mate 1's k-mers first, mate 2's k-mers that also occur in mate 1 skipped (:849-853).
 * Mate i of pair p = record p of buffer i; n_pairs = records zipped from the two files; n_bases_i = rec_off_i[n_pairs].  The reference's default
 * (approximate scalable cuckoo filter, fpr 1e-4) is not bit-reproducible and stays out of scope (SURVEY R11). */
int syl_sketch_read_pairs(syl_ctx *ctx, int mem, const uint8_t *bases1, uint64_t n_bases1, const uint64_t *rec_off1,
                          const uint8_t *bases2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                          int k, uint64_t c, int no_dedup, int sem, syl_sample **out);
/* The same for mates that are already 2-bit packed (layout: see syl_sketch_reads_packed2; one word buffer per mate file,
 * ceil(n_bases_i/16) words, rec_off_i in bases).  Same result as syl_sketch_read_pairs on the ASCII it was packed from.
 * SYL_MEM_HOST copies each word buffer and each offset array to the device once (4x fewer bytes than ASCII);
 * SYL_MEM_DEVICE word buffers must be 16-byte aligned (else SYL_ERR_ARG). */
int syl_sketch_read_pairs_packed2(syl_ctx *ctx, int mem, const uint32_t *packed1, uint64_t n_bases1, const uint64_t *rec_off1,
                                  const uint32_t *packed2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                                  int k, uint64_t c, int no_dedup, int sem, syl_sample **out);
/* Host-side packer used by the above: exact BYTE_TO_SEQ codes, n_threads <= 0 = default. */
int syl_pack2(const uint8_t *bases, uint64_t n_bases, uint32_t *words, int n_threads);
/* Worker threads the host-memory path of syl_sketch_reads packs with (for bench.py's e2e record). */
int syl_pack_threads(void);
/* What the last syl_sketch_reads(SYL_MEM_HOST, ASCII) call of this ctx moved: host-to-device bytes (bases + record
 * offsets, as copied) and how many of its chunks crossed the link as 2-bit words / as ASCII. */
int syl_ctx_ingest_stats(const syl_ctx *ctx, uint64_t *h2d_bytes, uint64_t *chunks_packed, uint64_t *chunks_ascii);
/* Wrap an existing sketch (e.g. a deserialised .sylsp).  Pairs need not be sorted; hashes must
 * be distinct. */
int syl_sample_upload(syl_ctx *ctx, int mem, const uint64_t *hash, const uint32_t *count,
                      uint64_t n, int k, uint64_t c, syl_sample **out);
uint64_t syl_sample_size(const syl_sample *s);
/* sum of rec lengths / n_reads (the reference keeps a running f64 mean, src/sketch.rs:941-943;
 * equal up to rounding, only feeds `-u` and `inspect`). */
double syl_sample_mean_read_length(const syl_sample *s);
uint64_t syl_sample_num_dup_removed(const syl_sample *s);
/* mean_read_length of an uploaded sketch (a .sylsp carries it; `-u` reads it, src/contain.rs:295) */
void syl_sample_set_mean_read_length(syl_sample *s, double mean_read_length);
int syl_sample_download(syl_ctx *ctx, const syl_sample *s, uint64_t *hash, uint32_t *count);
/* Raw device pointers (valid until syl_sample_free), for zero-copy interop. */
int syl_sample_device_ptrs(const syl_sample *s, const uint64_t **hash, const uint32_t **count);
void syl_sample_free(syl_sample *s);

/* ------------------------------------------------------------------------------------------
 * (3) Genome sketches — replaces sketch_genome (src/sketch.rs:550-622) / with individual != 0
 *     sketch_genome_individual (:481-548) for a batch of genomes whose contigs are already in
 *     a flat buffer.  genome_off[g]..genome_off[g+1] indexes contigs (records) of genome g.
 *     Result: CSR genome_kmers (position order) + CSR pseudotax_tracked_nonused_kmers +
 *     gn_size per genome (src/types.rs:163-173), resident on the device.
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_genomes syl_genomes;

int syl_sketch_genomes(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                       const uint64_t *contig_off, uint64_t n_contigs, const uint64_t *genome_off,
                       uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax,
                       int individual, int sem, syl_genomes **out);
/* The same for contigs that are already 2-bit packed (layout: see syl_sketch_reads_packed2; ceil(n_bases/16) words,
 * contig_off in bases): e.g. a 2-bit genome store.  Same result as syl_sketch_genomes on the ASCII it was packed
 * from (gn_size comes from contig_off).  SYL_MEM_HOST copies the words once (4x fewer bytes than ASCII);
 * SYL_MEM_DEVICE words must be 16-byte aligned (else SYL_ERR_ARG). */
int syl_sketch_genomes_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                               const uint64_t *contig_off, uint64_t n_contigs, const uint64_t *genome_off,
                               uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax,
                               int individual, int sem, syl_genomes **out);
/* Wrap existing sketches (e.g. a deserialised .syldb). tracked_off == NULL: no tracked k-mers (has_tracked = 0,
 * profile refuses the db); tracked may be NULL when tracked_off[n_genomes] == 0. */
int syl_genomes_upload(syl_ctx *ctx, int mem, const uint64_t *kmers, const uint64_t *kmer_off,
                       const uint64_t *tracked, const uint64_t *tracked_off, const uint64_t *gn_size,
                       uint64_t n_genomes, int k, uint64_t c, syl_genomes **out);
/* Concatenate batches (database build in chunks): genome i of part p becomes genome
 * (sum of earlier parts' counts) + i.  All parts must agree on k, c and has_tracked. */
int syl_genomes_concat(syl_ctx *ctx, const syl_genomes *const *parts, uint32_t n_parts, syl_genomes **out);
/* New batch holding genomes idx[0..n) of g (host index array), e.g. the pass-1 survivors of a
 * shard that are gathered into a small survivor database for the multi-GPU profile. */
int syl_genomes_select(syl_ctx *ctx, const syl_genomes *g, const uint32_t *idx, uint32_t n, syl_genomes **out);
uint64_t syl_genomes_count(const syl_genomes *g);
uint64_t syl_genomes_total_kmers(const syl_genomes *g);
uint64_t syl_genomes_total_tracked(const syl_genomes *g);
int syl_genomes_has_tracked(const syl_genomes *g);
int syl_genomes_k(const syl_genomes *g);
uint64_t syl_genomes_c(const syl_genomes *g);
/* Copy out: kmer_off/tracked_off have n_genomes+1 entries; any pointer may be NULL to skip. */
int syl_genomes_download(syl_ctx *ctx, const syl_genomes *g, uint64_t *kmers, uint64_t *kmer_off,
                         uint64_t *tracked, uint64_t *tracked_off, uint64_t *gn_size);
/* Raw device pointers of the CSR arrays (valid until syl_genomes_free), for zero-copy interop,
 * e.g. gathering survivor sketches across GPUs with NCCL. Any out pointer may be NULL. */
int syl_genomes_device_ptrs(const syl_genomes *g, const uint64_t **kmers, const uint64_t **kmer_off,
                            const uint64_t **tracked, const uint64_t **tracked_off, const uint64_t **gn_size);
void syl_genomes_free(syl_genomes *g);

/* ------------------------------------------------------------------------------------------
 * (4) Containment — replaces the pass-1 / pass-2 get_stats loops of contain()
 *     (src/contain.rs:284-292, 297-327) incl. ratio_lambda (src/inference.rs:207-242),
 *     ani_from_lambda (:817-847), bootstrap_interval (:849-898), winner_table (:410-430),
 *     derep_if_reassign_threshold (:353-375) and the abundance columns (:319-326).
 *
 * syl_db_build indexes a set of genome sketches for probing (one-time, amortised over samples).
 * genome_base is added to the genome index reported in result rows (multi-GPU shards).
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_db syl_db;

int syl_db_build(syl_ctx *ctx, const syl_genomes *g, uint32_t genome_base, syl_db **out);
uint64_t syl_db_num_genomes(const syl_db *db);
void syl_db_free(syl_db *db);

typedef struct {
    int32_t k;
    int32_t pseudotax;        /* 1 = `profile`, 0 = `query` */
    int32_t no_ci;            /* --no-ci */
    int32_t no_adj;           /* --no-adjust */
    int32_t mean_coverage;    /* --mean-coverage */
    int32_t estimate_unknown; /* -u: needs read_seq_id > 0 (the automatic identity estimate get_kmer_identity,
                                 src/contain.rs:901-951, walks a hash map in iteration order: SYL_ERR_UNSUPPORTED) */
    double min_number_kmers;  /* -M, default 50  (src/cmdline.rs:96) */
    double min_count_correct; /* default 3       (src/cmdline.rs:94) */
    double minimum_ani;       /* -m in percent; < 0 = unset => 90 (query) / 95 (profile) */
    double redundant_ani;     /* -R, default 99  (src/cmdline.rs:119) */
    double read_seq_id;       /* --read-seq-id in percent (src/contain.rs:274-277); <= 0 = unset */
} syl_contain_params;

void syl_contain_params_default(syl_contain_params *p, int k, int pseudotax);

enum { SYL_LAMBDA_LOW = 0, SYL_LAMBDA_HIGH = 1, SYL_LAMBDA_VALUE = 2 };

/* One AniResult (src/types.rs:185-204) minus the strings, 144 bytes. */
typedef struct {
    uint32_t sample;        /* index into the samples[] argument */
    uint32_t genome;        /* genome_base + index inside the db */
    uint32_t lambda_status; /* SYL_LAMBDA_* */
    uint32_t ci_valid;      /* 1 if the four CI values are Some */
    uint64_t contain;       /* containment_index.0 */
    uint64_t glen;          /* containment_index.1 */
    int64_t kmers_lost;     /* -1 = None (query) */
    double naive_ani;
    double final_est_ani;
    double final_est_cov;
    double mean_cov;        /* geq1_mean_cov */
    double median_cov;
    double lambda;          /* valid iff lambda_status == SYL_LAMBDA_VALUE */
    double ci[4];           /* ani 5%, ani 95%, lambda 5%, lambda 95% */
    double rel_abund;       /* profile only, else 0 */
    double seq_abund;       /* profile only, else 0 */
    double reserved;
} syl_ani_row;

/* Pass 1 only (== `query`, or the first half of `profile`): every (sample, genome) pair of
 * samples[] x db; rows only for pairs where get_stats returns Some. Rows are ordered by
 * (sample, genome).  rows: host buffer of cap entries. */
int syl_query(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
              const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);

/* Full `profile` for samples[] against ONE db holding all candidate genomes: pass 1, winner
 * table, pass 2, derep, abundances; rows sorted per sample by rel_abund descending
 * (src/contain.rs:329-334).  Ties in the winner table go to the lowest genome index (the
 * reference's tie winner is thread-timing dependent, SURVEY R10). */
int syl_profile(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);

/* ------------------------------------------------------------------------------------------
 * (5) `profile` over a genome-SHARDED database (one process per GPU; src/contain.rs:284-334 is the loop
 *     that is sharded).  Every rank holds a db built with its genome_base and ALL samples.  The library
 *     enqueues the compute stages on the ctx stream; the caller issues the three fixed-size collectives
 *     between them on the same stream (NCCL; no host synchronisation in between):
 *
 *       syl_profile_shard_begin      pass 1 on the shard -> d_table1 (header + rows_per_rank rows)
 *       all_gather(d_gathered1 <- d_table1)                         [world x table_bytes bytes]
 *       syl_profile_shard_rank       order of every pass-1 survivor; per sample key the best order
 *                                    among this shard's genomes -> d_winner (int32[winner_elems])
 *       all_reduce(d_winner, MIN)                                   [int32]
 *       syl_profile_shard_pass2      pass 2 (lost k-mers vs the global winner), bootstrap -> d_table2
 *       all_gather(d_gathered2 <- d_table2)
 *       syl_profile_shard_finish     the call's one host sync: derep, abundances, per-sample order; every
 *                                    rank returns the same rows (row.genome = global genome index)
 *
 *     rows_per_rank == 0 takes the default, 256 + 96 * n_samples rounded up to a multiple of 256 when world > 1:
 *     it does not depend on the shard, so every rank's table has the same size.  A rank whose shard holds no
 *     genome runs every stage (zeroed table headers, no winner candidates) and takes part in every collective.
 *     SYL_ERR_CAPACITY from finish: redo with rows_per_rank >= *need_rows_per_rank (same verdict on every
 *     rank).  SYL_ERR_UNSUPPORTED: a k-mer count >= 256 was met (every rank sees it); use the gathered-
 *     survivor path (sylph_b200/dist.py profile_sharded_gather).  world == 1 is allowed (no collectives).
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_profile_job syl_profile_job;
int syl_profile_shard_begin(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                            const syl_contain_params *p, uint32_t world, uint32_t rank, uint64_t rows_per_rank,
                            syl_profile_job **out);
int syl_profile_job_buffers(const syl_profile_job *job, void **d_table1, void **d_gathered1, uint64_t *table_bytes,
                            void **d_winner, uint64_t *winner_elems, void **d_table2, void **d_gathered2);
int syl_profile_shard_rank(syl_profile_job *job);
int syl_profile_shard_pass2(syl_profile_job *job);
int syl_profile_shard_finish(syl_profile_job *job, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows,
                             uint64_t *need_rows_per_rank);
void syl_profile_job_free(syl_profile_job *job);

#ifdef __cplusplus
}
#endif
#endif
