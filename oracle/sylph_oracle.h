/*
 * sylph_oracle.h — CPU restatement of sylph's two hot paths (TEST INFRASTRUCTURE ONLY).
 *
 * This is the parity oracle for sylph_b200.  It restates, in plain C, the algorithm of
 * bluenote-1577/sylph v0.8.1 (cited file:line relative to the root of the reference repository).
 * Nothing in the product path (sylph_b200/, include/) may include, link or call this file;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.
 *
 * PARITY PIN STATUS: the reference is a Rust crate and no Rust toolchain exists in the build
 * image, so the reference itself cannot be executed.  Its own tests hold no numeric golden
 * vectors (tests/integration_test.rs asserts exit codes / line counts only).  The oracle is
 * pinned on what does exist: (i) `profile o157_reads vs EC590` prints exactly 1 row
 * (tests/integration_test.rs:117-126), (ii) `query` vs EC590/o157/K12 prints exactly 3 rows
 * (:128-140), (iii) the scalar hash equals the AVX2 hash (tests/unit_test.rs:6,24), and it is
 * cross-checked by an independent pure-Python restatement (oracle/pyref.py).  Everything
 * else is "parity unpinned" by the reference: the third-party arithmetic (statrs Poisson CDF,
 * fastrand WyRand) is restated from the published algorithms of the pinned versions
 * (Cargo.lock: statrs 0.16.1, fastrand 2.1.1).
 */
#ifndef SYLPH_ORACLE_H
#define SYLPH_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Which window set a record contributes (src/sketch.rs:53-93 runtime dispatch). */
enum {
    SYO_SEM_SCALAR = 0, /* fmh_seeds: all L-k+1 windows            (src/seeding.rs:86-146)      */
    SYO_SEM_AVX2 = 1,   /* 4-lane split, trailing windows dropped  (src/avx2_seeding.rs:33-148) */
    SYO_SEM_AVX2_INTRIN = 2 /* same window set as SYO_SEM_AVX2, computed with AVX2 intrinsics (timed baseline) */
};

/* src/seeding.rs:4-15 (the shipped, "bugged" minimap2-style hash). */
uint64_t syo_mm_hash64(uint64_t kmer);
/* src/types.rs:50-59 */
uint8_t syo_byte_to_seq(uint8_t b);

/* extract_markers (src/sketch.rs:53-69).  Appends survivor hashes of one record to out (cap
 * entries available).  Returns the number of survivors (may exceed cap; only cap written). */
size_t syo_extract_markers(const uint8_t *s, size_t len, int k, uint64_t c, int sem,
                           uint64_t *out_hash, size_t cap);
/* extract_markers_positions (src/sketch.rs:71-93): also reports the end index of each window. */
size_t syo_extract_markers_positions(const uint8_t *s, size_t len, int k, uint64_t c, int sem,
                                     uint64_t *out_pos, uint64_t *out_hash, size_t cap);
/* Same as syo_extract_markers(…, SYO_SEM_AVX2) but written with AVX2 intrinsics so it does the
 * same per-base work as src/avx2_seeding.rs:33-148 (used for CPU-baseline timing). Requires
 * k in {21,31}. Returns (size_t)-1 when AVX2 is unavailable. */
size_t syo_extract_markers_avx2_intrin(const uint8_t *s, size_t len, int k, uint64_t c,
                                       uint64_t *out_hash, size_t cap);

/* sketch_genome (src/sketch.rs:550-622) over one genome given as concatenated contigs.
 * individual != 0 => sketch_genome_individual semantics for ONE record (src/sketch.rs:481-548).
 * out_kmers/out_tracked have cap entries each. Returns 0 ok, 1 if cap too small. */
int syo_sketch_genome(const uint8_t *bases, const uint64_t *contig_off, uint32_t n_contigs, int k,
                      uint64_t c, uint64_t min_spacing, int pseudotax, int sem,
                      uint64_t *out_kmers, size_t *n_kmers, uint64_t *out_tracked,
                      size_t *n_tracked, size_t cap, uint64_t *gn_size);

/* sketch_sequences_needle (src/sketch.rs:897-959) + dup_removal_lsh_full_exact (:690-731) +
 * pair_kmer_single (:624-656). Output sorted by hash. nthreads>1 parallelises only the seeding
 * (the dedup state machine stays sequential in file order). Returns 0 ok, 1 cap too small. */
int syo_sketch_reads(const uint8_t *bases, const uint64_t *rec_off, uint64_t n_reads, int k,
                     uint64_t c, int no_dedup, int sem, int nthreads, uint64_t *out_hash,
                     uint32_t *out_count, size_t *n_out, size_t cap, double *mean_read_length,
                     uint64_t *num_dup_removed);

/* src/sketch.rs:771-895 with dedup_fpr == 0 (exact pair set, no MAX_DEDUP_COUNT cap): mate files as two flat buffers */
int syo_sketch_read_pairs(const uint8_t *bases1, const uint64_t *off1, const uint8_t *bases2, const uint64_t *off2,
                          uint64_t n_pairs, int k, uint64_t c, int no_dedup, int sem, uint64_t *out_hash,
                          uint32_t *out_count, size_t *n_out, size_t cap, double *mean_read_length,
                          uint64_t *num_dup_removed);

/* ---- containment (src/contain.rs) ---- */
typedef struct {
    int k;
    double min_number_kmers;  /* src/cmdline.rs:96  default 50 */
    double min_count_correct; /* src/cmdline.rs:94  default 3  */
    double minimum_ani;       /* percent (0-100); < 0 => not set (src/contain.rs:746-748) */
    int pseudotax;            /* profile => 1 */
    int no_ci;
    int no_adj;
    int mean_coverage;
    double redundant_ani; /* src/cmdline.rs:119 default 99 */
} syo_params;

enum { SYO_LAMBDA_LOW = 0, SYO_LAMBDA_HIGH = 1, SYO_LAMBDA_VALUE = 2 };

typedef struct {
    uint32_t genome;      /* index into the db */
    uint32_t lambda_status;
    uint64_t contain;     /* containment_index.0 */
    uint64_t glen;        /* containment_index.1 = |genome_kmers| */
    int64_t kmers_lost;   /* -1 = None */
    double naive_ani;
    double final_est_ani;
    double final_est_cov;
    double mean_cov;      /* = geq1_mean_cov (src/contain.rs:789) */
    double median_cov;
    double lambda;        /* valid iff lambda_status == VALUE */
    double ci[4];         /* low_ani, high_ani, low_lambda, high_lambda */
    uint32_t ci_valid;    /* 1 if all four are Some */
    uint32_t pad;
    double rel_abund;     /* profile only */
    double seq_abund;     /* profile only */
} syo_ani_result;

typedef struct syo_sample syo_sample; /* FxHashMap<Kmer,u32> stand-in */
syo_sample *syo_sample_new(const uint64_t *hash, const uint32_t *count, size_t n);
void syo_sample_free(syo_sample *s);

/* get_stats pass 1 (winner_map = None) for one genome (src/contain.rs:601-814).
 * Returns 1 and fills *out if Some, 0 if None. */
int syo_get_stats(const syo_params *p, const uint64_t *genome_kmers, size_t n,
                  const syo_sample *sample, uint32_t genome_index, syo_ani_result *out);

/* Inner body of contain() for ONE sample against a CSR database (src/contain.rs:266-339):
 * pass 1 over all genomes; if p->pseudotax also winner_table (:410-430), pass 2 (:302-307),
 * derep_if_reassign_threshold (:353-375) and abundances (:319-326); final stable sort
 * (:329-334). Deterministic order: pass-1 results are taken in genome-index order (the
 * reference pushes them from rayon workers in timing-dependent order, SURVEY R10).
 * tracked_off/tracked may be NULL (db sketched with --disable-profiling).
 * out has cap rows; returns number of rows (or -1 if cap too small). */
/* -u / --estimate-unknown with --read-seq-id (percent): the sample's c and mean read length come from its sketch */
typedef struct { double read_seq_id; double mean_read_length; uint64_t sample_c; } syo_unknown;
int64_t syo_contain_sample(const syo_params *p, const uint64_t *kmers, const uint64_t *kmer_off,
                           const uint64_t *tracked, const uint64_t *tracked_off,
                           const uint64_t *gn_size, uint32_t n_genomes, const syo_sample *sample,
                           int nthreads, syo_ani_result *out, size_t cap);
int64_t syo_contain_sample_unknown(const syo_params *p, const uint64_t *kmers, const uint64_t *kmer_off,
                                   const uint64_t *tracked, const uint64_t *tracked_off,
                                   const uint64_t *gn_size, uint32_t n_genomes, const syo_sample *sample,
                                   int nthreads, syo_ani_result *out, size_t cap, const syo_unknown *u);

/* Largest cov with PoissonCDF(cov; median) < CUTOFF_PVALUE for median 1..29
 * (src/contain.rs:664-675, src/constants.rs:3) computed by direct summation. */
uint32_t syo_poisson_cutoff(uint32_t median);

/* fastrand 2.1.1 WyRand stream with seed s, n-th call of usize(..range) (1-based);
 * exposed so tests can pin the device's counter-based bootstrap RNG to it. */
uint64_t syo_fastrand_usize(uint64_t seed, uint64_t n_draw, uint64_t range);

/* TSV row text (src/contain.rs:18-94). Writes a NUL-terminated line (no newline) into buf. */
int syo_format_row(const syo_ani_result *r, int pseudotax, const char *seq_name,
                   const char *gn_name, const char *contig_name, char *buf, size_t buflen);

#ifdef __cplusplus
}
#endif
#endif
