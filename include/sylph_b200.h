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
 *     fewer than 2^32-2 survivor events per hash-range part of a read sample (section 2), fewer than 2^32-2 index entries (genome_kmers + tracked)
 *     and 2^31 genomes per db shard (a larger database from host memory: syl_db_shards, section 6), fewer than 2^31
 *     (sample, genome) pairs per syl_query / syl_profile call.
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

#define SYL_ABI_VERSION 3

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
    SYL_KERNEL_JOIN = 2,        /* containment pass 1: k_join_hist (+ k_range_bounds, CSR formulation: k_join2_order) */
    SYL_KERNEL_JOIN2 = 3,       /* containment pass 2: k_join2_order (+ k_local_best when sharded) */
    SYL_KERNEL_STATS = 4,       /* k_stats_hist / k_stats */
    SYL_KERNEL_BOOT = 5,        /* bootstrap: k_boot_iter_p (+ k_boot_seq, k_boot_final) */
    SYL_KERNEL_GENOME_POST = 6, /* genome-sketch post-pass (everything after k_seed) */
    SYL_KERNEL_PACK = 7,        /* ASCII -> 2-bit packing on the device (unused by the host-packed path) */
    SYL_KERNEL_SCAN = 8,        /* scan formulation of pass 1 (db shards): k_scan (+ the sample tables, k_table_*) */
    SYL_KERNEL_COUNT = 9
};
int syl_ctx_kernel_time(syl_ctx *ctx, int which, double *total_ms, uint64_t *launches, int reset);
/* Device memory of the ctx.  held: bytes of every block the ctx's block cache has allocated (blocks of live
 * sample / genomes / db handles and of profile jobs, plus cached free blocks; between calls nothing else is
 * allocated through it).  peak: high-water mark of held plus the live temporaries of syl_db_build /
 * syl_db_build_arrays since the ctx was created or the peak last reset (reset_peak != 0 resets it after reading).
 * The staging rings of the host-memory read and genome paths (syl_sketch_reads, syl_sketch_read_pairs and the genome
 * calls with SYL_MEM_HOST; syl_ctx_ingest_ring_bytes) are allocated directly and are not counted; the buffer of a
 * host genome larger than a chunk is a cached block and is. */
int syl_ctx_device_bytes(syl_ctx *ctx, uint64_t *held, uint64_t *peak, int reset_peak);

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
 * (approximate scalable cuckoo filter, fpr 1e-4) is not bit-reproducible and stays out of scope (SURVEY R11).
 * SYL_MEM_HOST: the sample crosses the link as chunks of pairs (both mates of a chunk 2-bit packed by the worker
 * threads into one pinned staging buffer, or shipped as ASCII: SYL_HOST_INGEST as for syl_sketch_reads) while earlier
 * chunks are seeded, so the device holds the staging rings and the events, never the sample's bases. */
int syl_sketch_read_pairs(syl_ctx *ctx, int mem, const uint8_t *bases1, uint64_t n_bases1, const uint64_t *rec_off1,
                          const uint8_t *bases2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                          int k, uint64_t c, int no_dedup, int sem, syl_sample **out);
/* The same for mates that are already 2-bit packed (layout: see syl_sketch_reads_packed2; one word buffer per mate file,
 * ceil(n_bases_i/16) words, rec_off_i in bases).  Same result as syl_sketch_read_pairs on the ASCII it was packed from.
 * SYL_MEM_HOST copies each word buffer and each offset array to the device whole, once (4x fewer bytes than ASCII; not chunked);
 * SYL_MEM_DEVICE word buffers must be 16-byte aligned (else SYL_ERR_ARG). */
int syl_sketch_read_pairs_packed2(syl_ctx *ctx, int mem, const uint32_t *packed1, uint64_t n_bases1, const uint64_t *rec_off1,
                                  const uint32_t *packed2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                                  int k, uint64_t c, int no_dedup, int sem, syl_sample **out);
/* Host-side packer used by the above: exact BYTE_TO_SEQ codes, n_threads <= 0 = default. */
int syl_pack2(const uint8_t *bases, uint64_t n_bases, uint32_t *words, int n_threads);
/* Worker threads the host-memory path of syl_sketch_reads packs with (for bench.py's e2e record). */
int syl_pack_threads(void);
/* What the last syl_sketch_reads / syl_sketch_read_pairs(SYL_MEM_HOST, ASCII) call or syl_sketch_genomes /
 * syl_sketch_genomes_packed2(SYL_MEM_HOST) call of this ctx moved: host-to-device bytes (bases or words + record
 * offsets, as copied; for genomes also every chunk's genome offsets) and how many of its chunks (of reads, of pairs,
 * of genomes) crossed the link as 2-bit words / as ASCII.  Host 2-bit reads and pairs are staged whole: their bytes,
 * no chunks.  A genome larger than a chunk counts as one chunk of the form it crossed in. */
int syl_ctx_ingest_stats(const syl_ctx *ctx, uint64_t *h2d_bytes, uint64_t *chunks_packed, uint64_t *chunks_ascii);
/* Bytes the host-memory staging rings of this ctx hold now: on the device (allocated outside the block cache, so
 * syl_ctx_device_bytes does not count them) and in pinned host memory.  Read and genome calls share them.  They grow
 * to the largest chunk seen (a genome larger than a chunk is staged in cached blocks instead, and does not grow them)
 * and live until the ctx is destroyed. */
int syl_ctx_ingest_ring_bytes(const syl_ctx *ctx, uint64_t *device_bytes, uint64_t *pinned_bytes);
/* Device memory of read and pair sketches (the four calls above).  The post-pass holds about 120 bytes per expected
 * survivor event (bases / c), and host input adds its staging rings or, for 2-bit words, the staged words.  A sample
 * whose one-pass estimate does not fit the budget is sketched in P parts (at most 64): contiguous hash ranges of
 * [0, 2^64 / c), each in a pass of its own over the input (device input read in place, host 2-bit words staged once,
 * host ASCII fed again for every part).  The parts' sketches wait in host memory and are assembled into the same
 * sketch, num_dup_removed and mean_read_length as one pass gives.  A budget that even 64 parts exceed is SYL_ERR_OOM
 * before anything is allocated; the message names the bytes needed.
 * syl_ctx_set_sample_memory: max_bytes of device memory a sketch call may use (block-cache blocks plus staging rings),
 *   and that a host-samples query or profile (section 7) may use in block-cache blocks (its batch slots, sort and join
 *   scratch, and with shards the largest shard's build; the staging rings, which that call shares with the sketch
 *   calls and leaves allocated, are not counted against it);
 *   0 (the default) = the device's free memory at call time plus what the ctx holds in cached free blocks and rings
 *   (a sample whose one pass needs less than half of the free memory the ctx saw at its last look takes one pass
 *   without looking again).
 * syl_ctx_sample_memory: the budget set (0: default) and the device's free memory now (either pointer may be NULL),
 *   e.g. to split one device between several contexts.
 * syl_ctx_sample_parts: P of the last read or pair sketch of this ctx (1: one pass).
 * SYL_SAMPLE_PARTS=N (test hook, read per call) forces N parts, at most one per post-pass bucket. */
int syl_ctx_set_sample_memory(syl_ctx *ctx, uint64_t max_bytes);
int syl_ctx_sample_memory(syl_ctx *ctx, uint64_t *max_bytes, uint64_t *free_bytes);
int syl_ctx_sample_parts(const syl_ctx *ctx, uint32_t *parts);
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
 *     SYL_MEM_HOST: the batch crosses the link in chunks of whole genomes (whole contigs with individual != 0) of at most
 *     the read path's chunk size and 2^19 contigs, through the staging rings of syl_sketch_reads (ASCII packed to 2 bits
 *     by the worker threads or shipped as it is, SYL_HOST_INGEST as there; 2-bit words copied as they are), while
 *     earlier chunks are sketched.  A genome larger than a chunk is copied on its own into one buffer as large as the
 *     genome.  Each chunk is sketched with its genomes' survivors alone (the post-pass needs nothing else), and the
 *     chunks' results are joined in order into one handle, the same as from device memory.  The device holds the output
 *     (about 8 bytes per kept or tracked k-mer) twice at most, one chunk's working set (about 1.5 bytes per base of the
 *     chunk) and the rings, never the batch's bases; the 2^32-2 survivor limit applies per chunk.
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_genomes syl_genomes;

int syl_sketch_genomes(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                       const uint64_t *contig_off, uint64_t n_contigs, const uint64_t *genome_off,
                       uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax,
                       int individual, int sem, syl_genomes **out);
/* The same for contigs that are already 2-bit packed (layout: see syl_sketch_reads_packed2; ceil(n_bases/16) words,
 * contig_off in bases): e.g. a 2-bit genome store.  Same result as syl_sketch_genomes on the ASCII it was packed
 * from (gn_size comes from contig_off).  SYL_MEM_HOST copies each chunk's words (4x fewer bytes than ASCII) from the
 * word of its first base, with no packing, into a ring slot; pageable words are copied chunk by chunk too.
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
/* The same index straight from CSR arrays in host or device memory (e.g. a deserialised .syldb), without a
 * syl_genomes: arguments as in syl_genomes_upload (tracked_off == NULL: no tracked k-mers, profile refuses the db;
 * gn_size may be NULL: zeros).  Offsets must start at 0 and be monotone, k-mers plus tracked k-mers must stay below
 * 2^32 - 2 and genomes below 2^31 - 1 (else SYL_ERR_ARG, before anything is allocated).  The build holds the index
 * (12 bytes per entry), the bucket directory (4 bytes per bucket, about one per 2-4 entries) and 4 bytes per genome,
 * plus temporaries it frees before returning: from host memory two staging chunks of SYL_DB_CHUNK entries each
 * (default 2^25; 8 bytes per entry plus 16 per genome up to the chunk size), and for buckets of more than 2048 entries
 * (a key shared by that many genomes) about 16 bytes per entry of the largest one.  Host input is read three times,
 * chunk by chunk, each chunk copied straight from the arrays on the ctx's copy stream (the one its host-memory staging
 * shares; no staging ring is allocated) while the previous one is processed. */
int syl_db_build_arrays(syl_ctx *ctx, int mem, const uint64_t *kmers, const uint64_t *kmer_off, const uint64_t *tracked,
                        const uint64_t *tracked_off, const uint64_t *gn_size, uint64_t n_genomes, int k, uint64_t c,
                        uint32_t genome_base, syl_db **out);
/* Copy the index out to host memory: keys[n_entries] ascending, gid[n_entries] = genome << 1 | tracked (entries of
 * one key ordered by tracked, then genome), bstart[n_buckets + 1] bucket starts.  Array pointers may be NULL, so a
 * call with NULL arrays only reports the sizes. */
int syl_db_download(syl_ctx *ctx, const syl_db *db, uint64_t *keys, uint32_t *gid, uint32_t *bstart, uint64_t *n_entries,
                    uint64_t *n_buckets);
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
 *
 *     Each rank picks its own join formulation in begin: the per-pair count histograms, or the CSR formulation
 *     when csr != 0, when SYL_CONTAIN_CSR is set or when its shard's histograms would exceed 8 GB (samples x
 *     shard genomes > 2^23 pairs).  Both write the same row tables, so ranks may run different formulations.
 *     CSR adds one host synchronisation inside begin, before the first collective.
 *
 *     SYL_ERR_CAPACITY from finish: redo with rows_per_rank >= *need_rows_per_rank.  SYL_ERR_UNSUPPORTED from
 *     finish: a histogram rank met a k-mer count >= 256; redo the job with csr = 1.  Both verdicts come from the
 *     gathered table headers, so every rank reaches the same one.  world == 1 is allowed (no collectives).
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_profile_job syl_profile_job;
int syl_profile_shard_begin(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                            const syl_contain_params *p, uint32_t world, uint32_t rank, uint64_t rows_per_rank,
                            int csr, syl_profile_job **out);
int syl_profile_job_buffers(const syl_profile_job *job, void **d_table1, void **d_gathered1, uint64_t *table_bytes,
                            void **d_winner, uint64_t *winner_elems, void **d_table2, void **d_gathered2);
int syl_profile_shard_rank(syl_profile_job *job);
int syl_profile_shard_pass2(syl_profile_job *job);
int syl_profile_shard_finish(syl_profile_job *job, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows,
                             uint64_t *need_rows_per_rank);
void syl_profile_job_free(syl_profile_job *job);

/* ------------------------------------------------------------------------------------------
 * (6) A database larger than one index, on ONE GPU, from host memory: e.g. GTDB at a small c, or several .syldb
 *     profiled together (sylph keeps the whole database in host RAM, src/contain.rs:212-236).  The 2^32-2 entry
 *     limit and the device memory then bound each shard, not the database.
 *
 * syl_db_shards_create borrows CSR arrays in HOST memory (arguments as in syl_db_build_arrays; the caller keeps them
 * alive and unchanged until syl_db_shards_free) and cuts them into contiguous genome ranges of at most max_entries
 * index entries (k-mers + tracked k-mers) each, greedily in genome order.  max_entries == 0: the largest shard the
 * device's free memory allows at creation (16 bytes per entry after 4 GB and an eighth of it for the joins); never
 * more than 2^32-3 entries or 2^31-2 genomes.  A genome larger than the cap is a shard of its own.  NULL arrays that
 * the offsets say hold entries, offsets that do not start at 0 or decrease, device pointers, 2^32 genomes or more, and
 * a genome of more than 2^32-3 entries are SYL_ERR_ARG, before anything is allocated.  Nothing is built yet.
 * SYL_DB_SHARD_ENTRIES (test hook, read per create) caps max_entries further.
 *
 * syl_query_shards / syl_profile_shards return the rows, order and error codes of syl_query / syl_profile on one db
 * of all genomes; row.genome is the global genome index.  Each call sweeps the shards once: it builds a shard's
 * index (as syl_db_build_arrays, genome_base = the shard's first genome), runs pass 1 of all samples against it in
 * batches of at most 2^22 (sample, genome) pairs, and frees it before building the next.  A call therefore costs one
 * index build per shard, whatever the sample count: give it all samples at once.  Device memory peaks at one shard's
 * build (see syl_db_build_arrays) plus the joins' scratch; the ctx's cached free blocks are released between shards.
 *   query:   rows ordered by (sample, genome).
 *   profile: pass 1 without CIs, then for each batch of samples an index of the union of their pass-1 survivors
 *            (ascending global order, gathered into pinned host staging) and syl_profile on it.  A batch closes before
 *            its union passes the shard cap; one sample's survivors may take up to max(cap, the free-memory default)
 *            entries, beyond that SYL_ERR_UNSUPPORTED.
 * SYL_ERR_CAPACITY: *n_rows holds the needed size, and the handle keeps the rows.  The NEXT call on the handle with the
 * same samples (pointers), params and kind only copies them out (no index is built); any other call drops them.
 * One ctx per handle; calls on one handle are serialised by the caller.
 * ---------------------------------------------------------------------------------------- */
typedef struct syl_db_shards syl_db_shards;
int syl_db_shards_create(syl_ctx *ctx, const uint64_t *kmers, const uint64_t *kmer_off, const uint64_t *tracked,
                         const uint64_t *tracked_off, const uint64_t *gn_size, uint64_t n_genomes, int k, uint64_t c,
                         uint64_t max_entries, syl_db_shards **out);
uint64_t syl_db_shards_count(const syl_db_shards *s);
/* shard i: genomes [*first_genome, *first_genome + *n_genomes) holding *n_entries index entries (out pointers may be NULL) */
int syl_db_shards_range(const syl_db_shards *s, uint64_t i, uint64_t *first_genome, uint64_t *n_genomes, uint64_t *n_entries);
int syl_query_shards(syl_ctx *ctx, syl_db_shards *s, const syl_sample *const *samples, uint32_t n_samples,
                     const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);
int syl_profile_shards(syl_ctx *ctx, syl_db_shards *s, const syl_sample *const *samples, uint32_t n_samples,
                       const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);
void syl_db_shards_free(syl_db_shards *s);
/* Scan instead of build.  A call of few samples on a large syl_db_shards handle does not build any index: its pass 1
 * streams the genome k-mers (never the tracked ones) from the borrowed host arrays to the device in chunks of whole
 * genomes, on the ctx's copy stream (pageable arrays through its pinned ring) into two device buffers,
 * chunk i + 1 while chunk i is scanned, and every genome k-mer probes a lookup table of every sample (about 6 bytes of
 * device memory per sample k-mer).  The rows, their order and the capacity protocol are those of the build path,
 * bit for bit; profile's pass 2 runs on the survivor indexes as above.  A call scans when all its samples fit one
 * sample batch, the database holds at least 2^28 index entries, and the measured cost model of DESIGN.md §10 puts
 * the scan below the build (it depends on whether the genome k-mers are in pinned memory, and on whether all samples'
 * tables fit the L2 cache).  SYL_DB_SCAN=0|1 (read per call) forces the build or the scan, the scan only where the
 * samples fit one batch (host samples that do not are swept shard by shard, as without the switch);
 * SYL_DB_SCAN_CHUNK=N (test hook, read per call) sets the genome k-mers per chunk (default 2^25).
 * syl_db_scan_plan sets *scan to what a call of n_samples samples holding sample_kmers k-mers together would do on a
 * handle of n_genomes genomes holding n_kmers genome k-mers and n_tracked tracked k-mers (1: scan, 0: build), taking
 * the samples as equal host samples for the batch condition and the database as pageable host arrays. */
int syl_db_scan_plan(syl_ctx *ctx, uint64_t n_kmers, uint64_t n_tracked, uint64_t n_genomes, uint32_t n_samples,
                     uint64_t sample_kmers, int *scan);

/* ------------------------------------------------------------------------------------------
 * (7) Query and profile samples from HOST memory, any number of them, in bounded device memory: e.g. every deserialised
 *     .sylsp of a study (the reference reads, sketches and profiles samples one chunk at a time, src/contain.rs:239-269).
 *
 * syl_host_samples: sample i holds the pairs hash[off[i] .. off[i + 1]) / count[...], in any order (as a .sylsp map),
 * with distinct hashes; c[i] and mean_read_length[i] are its sketch parameter and mean read length (-u reads it); k is
 * every sample's.  The arrays are borrowed for the duration of the call, in pinned or pageable host memory.
 *
 * syl_query_host_samples / syl_profile_host_samples take exactly one of db or shards (else SYL_ERR_ARG) and return the
 * rows, order and values of syl_query / syl_profile (syl_query_shards / syl_profile_shards) on handles made with
 * syl_sample_upload + syl_sample_set_mean_read_length from the same arrays; row.sample is the index into s.  The
 * arguments are checked as there, before anything is allocated; offsets that do not start at 0 or decrease and device
 * pointers are SYL_ERR_ARG.  SYL_ERR_CAPACITY: with a db, resize and call again; with shards, the handle keeps the rows
 * as in section (6), keyed on the array pointers and n_samples.
 *
 * The samples are cut into contiguous batches, each the longest run that fits half the device budget of
 * syl_ctx_set_sample_memory and at most 2^22 (sample, genome) pairs (with shards: pairs of the largest shard).  A batch
 * costs its slot (12 bytes per k-mer), its share of the sort's second buffer (24 bytes per k-mer over both slots) and
 * its joins' scratch (about 1 KB per pair, 16 bytes per k-mer of its largest sample per sample, 200 KB per sample);
 * with shards the budget also covers the largest shard's build (16 bytes per entry).  The default budget is the free
 * memory once the ctx's staging ring exists, plus the ctx's cached free blocks.  A sample that does not fit alone
 * is SYL_ERR_OOM before anything is allocated, with the bytes it needs in the message.  The joins' allocations the plan
 * does not charge (the CSR formulation's 4 bytes per hit, the row tables of samples with more than 96 rows) are held to
 * the budget on top of what the ctx held in use when the call began: a batch whose joins would pass it is rerun as two
 * halves, recursively, with the same rows, and a sample that does not fit alone is SYL_ERR_OOM, naming its bytes.
 * Each batch crosses the link in one pass on the ctx's copy stream (pageable arrays through its pinned
 * ring) and is sorted there by one segmented sort, while the previous batch is joined on the ctx stream.  With shards, each shard is built once per
 * call: every batch is joined with it before the next one is built (profile: then its survivor indexes, each joined
 * with samples of one batch, staged again unless a slot still holds them, while the index is gathered and built).
 * SYL_SAMPLE_BATCH=N (test hook, read per call) caps a batch at N samples.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    const uint64_t *hash;            /* all samples' k-mers back to back */
    const uint32_t *count;
    const uint64_t *off;             /* n_samples + 1 monotone offsets, off[0] == 0 */
    const uint64_t *c;               /* per sample */
    const double *mean_read_length;  /* per sample */
    uint32_t n_samples;
    int k;
} syl_host_samples;

int syl_query_host_samples(syl_ctx *ctx, const syl_db *db, syl_db_shards *shards, const syl_host_samples *s,
                           const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);
int syl_profile_host_samples(syl_ctx *ctx, const syl_db *db, syl_db_shards *shards, const syl_host_samples *s,
                             const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows);

#ifdef __cplusplus
}
#endif
#endif
