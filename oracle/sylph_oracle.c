/*
 * sylph_oracle.c — CPU restatement of sylph v0.8.1's sketch + containment hot paths.
 * TEST INFRASTRUCTURE ONLY (see sylph_oracle.h for the usage rule and the parity-pin status).
 * Every function cites the reference file:line (relative to the root of the reference repository) it follows.
 */
#include "sylph_oracle.h"

#include <math.h>
#include <quadmath.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#if defined(__x86_64__)
#include <immintrin.h>
#endif

/* ------------------------------------------------------------------------------------------
 * L0: alphabet + hash
 * ---------------------------------------------------------------------------------------- */

/* src/types.rs:50-59 — BYTE_TO_SEQ. Only A/C/G/T/U (either case) and the raw bytes 1..3 map to
 * a non-zero code; every other byte (N included) is 0, i.e. 'A'. */
uint8_t syo_byte_to_seq(uint8_t b) {
    switch (b) {
    case 1: case 'C': case 'c': return 1;
    case 2: case 'G': case 'g': return 2;
    case 3: case 'T': case 't': case 'U': case 'u': return 3;
    default: return 0;
    }
}

static uint8_t g_lut[256];
static int g_lut_ready = 0;
static const uint8_t *lut(void) {
    if (!g_lut_ready) {
        for (int i = 0; i < 256; i++) g_lut[i] = syo_byte_to_seq((uint8_t)i);
        g_lut_ready = 1;
    }
    return g_lut;
}

/* src/seeding.rs:4-15. Note line 7: `!key.wrapping_add(key << 21)` negates the SUM (method
 * call binds tighter than unary !), unlike minimap2's (~key) + (key << 21). */
uint64_t syo_mm_hash64(uint64_t key) {
    key = ~(key + (key << 21));
    key = key ^ (key >> 24);
    key = (key + (key << 3)) + (key << 8);
    key = key ^ (key >> 14);
    key = (key + (key << 2)) + (key << 4);
    key = key ^ (key >> 28);
    key = key + (key << 31);
    return key;
}

/* ------------------------------------------------------------------------------------------
 * L1: FracMinHash seeding
 * ---------------------------------------------------------------------------------------- */

typedef struct {
    uint64_t *pos;  /* may be NULL */
    uint64_t *hash; /* may be NULL when cap == 0 */
    size_t cap, n;
} emit_t;

static inline void emit(emit_t *e, uint64_t pos, uint64_t h) {
    if (e->n < e->cap) {
        if (e->pos) e->pos[e->n] = pos;
        e->hash[e->n] = h;
    }
    e->n++;
}

/* src/seeding.rs:86-146 (fmh_seeds) and :148-209 (fmh_seeds_positions): same loop, the latter
 * also reports i (index of the window's last base). */
static void seeds_scalar(const uint8_t *s, size_t len, size_t k, uint64_t c, emit_t *e) {
    if (len < k) return;
    const uint8_t *L = lut();
    uint64_t f = 0, r = 0;
    const unsigned rshift = (unsigned)(2 * (k - 1));
    const uint64_t mask = UINT64_MAX >> (64 - 2 * k);
    const uint64_t rev_mask = ~((uint64_t)3 << (2 * k - 2));
    const uint64_t thr = UINT64_MAX / c;
    for (size_t i = 0; i + 1 < k; i++) {
        uint64_t nf = L[s[i]], nr = 3 - nf;
        f = (f << 2) | nf;
        r = (r >> 2) | (nr << rshift);
    }
    for (size_t i = k - 1; i < len; i++) {
        uint64_t nf = L[s[i]], nr = 3 - nf;
        f = ((f << 2) | nf) & mask;
        r = ((r >> 2) & rev_mask) | (nr << rshift);
        uint64_t canon = (f < r) ? f : r;
        uint64_t h = syo_mm_hash64(canon);
        if (h < thr) emit(e, i, h);
    }
}

/* src/avx2_seeding.rs:33-148 / :151-266 restated lane by lane in scalar C.  The sequence is cut
 * into 4 lanes of lenq = (L-k+1)/4 windows; lane j sees string[j*lenq .. (j+1)*lenq + k-1) and
 * rolls independently; windows >= 4*lenq are never visited.  Survivors are pushed i-major,
 * lane-minor (:133-144).  min_len is k+1 for the hash-only variant (:42-44) and 2k for the
 * positions variant (:160-162).  k must be 21 or 31 (:46-52 panics otherwise). */
static int seeds_avx2sem(const uint8_t *s, size_t len, size_t k, uint64_t c, size_t min_len,
                         emit_t *e) {
    if (len < k) return 0;
    if (len < min_len) return 0;
    if (!(k == 21 || k == 31)) return -1;
    const uint8_t *L = lut();
    const size_t lenq = (len - k + 1) / 4;
    const unsigned rshift = (unsigned)(2 * (k - 1));
    const uint64_t mask = UINT64_MAX >> (64 - 2 * k);
    const uint64_t rev_mask = ~((uint64_t)3 << (2 * k - 2));
    const uint64_t thr = UINT64_MAX / c;
    uint64_t f[4] = {0, 0, 0, 0}, r[4] = {0, 0, 0, 0};
    for (size_t i = 0; i + 1 < k; i++) {
        for (int j = 0; j < 4; j++) {
            uint64_t nf = L[s[(size_t)j * lenq + i]], nr = 3 - nf;
            f[j] = (f[j] << 2) | nf;
            r[j] = (r[j] >> 2) | (nr << rshift);
        }
    }
    for (size_t i = k - 1; i < lenq + k - 1; i++) {
        for (int j = 0; j < 4; j++) {
            uint64_t nf = L[s[(size_t)j * lenq + i]], nr = 3 - nf;
            f[j] = ((f[j] << 2) | nf) & mask;
            r[j] = ((r[j] >> 2) & rev_mask) | (nr << rshift);
            /* cmpgt(r,f) ? f : r  (:121-124); values < 2^62 so signed == unsigned */
            uint64_t canon = (r[j] > f[j]) ? f[j] : r[j];
            uint64_t h = syo_mm_hash64(canon);
            if (h < thr) emit(e, (uint64_t)j * lenq + i, h);
        }
    }
    return 0;
}

size_t syo_extract_markers(const uint8_t *s, size_t len, int k, uint64_t c, int sem,
                           uint64_t *out_hash, size_t cap) {
    emit_t e = {NULL, out_hash, cap, 0};
    if (sem == SYO_SEM_AVX2_INTRIN) return syo_extract_markers_avx2_intrin(s, len, k, c, out_hash, cap);
    if (sem == SYO_SEM_SCALAR) {
        seeds_scalar(s, len, (size_t)k, c, &e);
    } else {
        if (seeds_avx2sem(s, len, (size_t)k, c, (size_t)k + 1, &e) < 0) return (size_t)-1;
    }
    return e.n;
}

size_t syo_extract_markers_positions(const uint8_t *s, size_t len, int k, uint64_t c, int sem,
                                     uint64_t *out_pos, uint64_t *out_hash, size_t cap) {
    emit_t e = {out_pos, out_hash, cap, 0};
    if (sem == SYO_SEM_SCALAR) {
        seeds_scalar(s, len, (size_t)k, c, &e);
    } else {
        if (seeds_avx2sem(s, len, (size_t)k, c, 2 * (size_t)k, &e) < 0) return (size_t)-1;
    }
    return e.n;
}

#if defined(__x86_64__)
/* src/avx2_seeding.rs:6-30 */
__attribute__((target("avx2"))) static inline __m256i hash256(__m256i key) {
    key = _mm256_add_epi64(key, _mm256_slli_epi64(key, 21));
    key = _mm256_xor_si256(key, _mm256_set1_epi64x(-1));
    key = _mm256_xor_si256(key, _mm256_srli_epi64(key, 24));
    key = _mm256_add_epi64(_mm256_add_epi64(key, _mm256_slli_epi64(key, 3)),
                           _mm256_slli_epi64(key, 8));
    key = _mm256_xor_si256(key, _mm256_srli_epi64(key, 14));
    key = _mm256_add_epi64(_mm256_add_epi64(key, _mm256_slli_epi64(key, 2)),
                           _mm256_slli_epi64(key, 4));
    key = _mm256_xor_si256(key, _mm256_srli_epi64(key, 28));
    key = _mm256_add_epi64(key, _mm256_slli_epi64(key, 31));
    return key;
}

/* src/avx2_seeding.rs:33-148 with intrinsics: per base 4 scalar LUT loads + set_epi64x, vector
 * roll / canonical / hash, then 4 scalar extract+compare — the same work the reference does, so
 * this is the timed CPU baseline kernel. */
__attribute__((target("avx2"))) static size_t seeds_avx2_intrin(const uint8_t *s, size_t len,
                                                                size_t k, uint64_t c,
                                                                uint64_t *out, size_t cap) {
    if (len < k || len < k + 1) return 0;
    const uint8_t *L = lut();
    const size_t lenq = (len - k + 1) / 4;
    const uint8_t *s0 = s, *s1 = s + lenq, *s2 = s + 2 * lenq, *s3 = s + 3 * lenq;
    const int rsh = (int)(2 * (k - 1));
    const __m128i rcount = _mm_cvtsi32_si128(rsh);
    const __m256i three = _mm256_set1_epi64x(3);
    const __m256i vmask = _mm256_set1_epi64x((long long)(UINT64_MAX >> (64 - 2 * k)));
    const __m256i vrmask = _mm256_set1_epi64x((long long)~((uint64_t)3 << (2 * k - 2)));
    const uint64_t thr = UINT64_MAX / c;
    __m256i f = _mm256_setzero_si256(), r = _mm256_setzero_si256();
    size_t n = 0;
    for (size_t i = 0; i + 1 < k; i++) {
        __m256i nf = _mm256_set_epi64x(L[s3[i]], L[s2[i]], L[s1[i]], L[s0[i]]);
        __m256i nr = _mm256_sub_epi64(three, nf);
        f = _mm256_or_si256(_mm256_slli_epi64(f, 2), nf);
        r = _mm256_or_si256(_mm256_srli_epi64(r, 2), _mm256_sll_epi64(nr, rcount));
    }
    for (size_t i = k - 1; i < lenq + k - 1; i++) {
        __m256i nf = _mm256_set_epi64x(L[s3[i]], L[s2[i]], L[s1[i]], L[s0[i]]);
        __m256i nr = _mm256_sub_epi64(three, nf);
        f = _mm256_and_si256(_mm256_or_si256(_mm256_slli_epi64(f, 2), nf), vmask);
        r = _mm256_or_si256(_mm256_and_si256(_mm256_srli_epi64(r, 2), vrmask),
                            _mm256_sll_epi64(nr, rcount));
        __m256i gt = _mm256_cmpgt_epi64(r, f);
        __m256i canon = _mm256_blendv_epi8(r, f, gt);
        __m256i h = hash256(canon);
        uint64_t v0 = (uint64_t)_mm256_extract_epi64(h, 0);
        uint64_t v1 = (uint64_t)_mm256_extract_epi64(h, 1);
        uint64_t v2 = (uint64_t)_mm256_extract_epi64(h, 2);
        uint64_t v3 = (uint64_t)_mm256_extract_epi64(h, 3);
        if (v0 < thr) { if (n < cap) out[n] = v0; n++; }
        if (v1 < thr) { if (n < cap) out[n] = v1; n++; }
        if (v2 < thr) { if (n < cap) out[n] = v2; n++; }
        if (v3 < thr) { if (n < cap) out[n] = v3; n++; }
    }
    return n;
}
#endif

size_t syo_extract_markers_avx2_intrin(const uint8_t *s, size_t len, int k, uint64_t c,
                                       uint64_t *out_hash, size_t cap) {
#if defined(__x86_64__)
    if (!__builtin_cpu_supports("avx2")) return (size_t)-1;
    if (!(k == 21 || k == 31)) return (size_t)-1;
    return seeds_avx2_intrin(s, len, (size_t)k, c, out_hash, cap);
#else
    (void)s; (void)len; (void)k; (void)c; (void)out_hash; (void)cap;
    return (size_t)-1;
#endif
}

/* ------------------------------------------------------------------------------------------
 * small open-addressing containers (stand-ins for FxHashMap / FxHashSet / MMHashSet; only
 * membership semantics are observable, never iteration order)
 * ---------------------------------------------------------------------------------------- */

#define EMPTY_KEY UINT64_MAX /* hashes are < u64::MAX/c <= u64::MAX, so never a valid key */

static inline uint64_t mix(uint64_t x) {
    x ^= x >> 31;
    x *= 0x9E3779B97F4A7C15ull;
    x ^= x >> 29;
    return x;
}

typedef struct {
    uint64_t *keys;
    uint32_t *vals;
    size_t capmask, n;
} u64map;

static void u64map_init(u64map *m, size_t expect) {
    size_t cap = 16;
    while (cap < expect * 2 + 2) cap <<= 1;
    m->keys = (uint64_t *)malloc(cap * sizeof(uint64_t));
    m->vals = (uint32_t *)calloc(cap, sizeof(uint32_t));
    for (size_t i = 0; i < cap; i++) m->keys[i] = EMPTY_KEY;
    m->capmask = cap - 1;
    m->n = 0;
}
static void u64map_free(u64map *m) { free(m->keys); free(m->vals); }
static uint32_t *u64map_find(const u64map *m, uint64_t key) {
    size_t i = mix(key) & m->capmask;
    while (m->keys[i] != EMPTY_KEY) {
        if (m->keys[i] == key) return &m->vals[i];
        i = (i + 1) & m->capmask;
    }
    return NULL;
}
static void u64map_grow(u64map *m);
/* entry(key).or_insert(0) */
static uint32_t *u64map_entry(u64map *m, uint64_t key) {
    if ((m->n + 1) * 2 > m->capmask + 1) u64map_grow(m);
    size_t i = mix(key) & m->capmask;
    while (m->keys[i] != EMPTY_KEY) {
        if (m->keys[i] == key) return &m->vals[i];
        i = (i + 1) & m->capmask;
    }
    m->keys[i] = key;
    m->vals[i] = 0;
    m->n++;
    return &m->vals[i];
}
static void u64map_grow(u64map *m) {
    u64map o = *m;
    size_t cap = (o.capmask + 1) * 2;
    m->keys = (uint64_t *)malloc(cap * sizeof(uint64_t));
    m->vals = (uint32_t *)calloc(cap, sizeof(uint32_t));
    for (size_t i = 0; i < cap; i++) m->keys[i] = EMPTY_KEY;
    m->capmask = cap - 1;
    m->n = 0;
    for (size_t i = 0; i <= o.capmask; i++)
        if (o.keys[i] != EMPTY_KEY) *u64map_entry(m, o.keys[i]) = o.vals[i];
    u64map_free(&o);
}

/* FxHashSet<(u64,[u32;2])> (src/sketch.rs:692) */
typedef struct { uint64_t km; uint32_t a, b; } pairkey;
typedef struct {
    pairkey *e;
    size_t capmask, n;
} pairset;
static void pairset_init(pairset *s, size_t expect) {
    size_t cap = 16;
    while (cap < expect * 2 + 2) cap <<= 1;
    s->e = (pairkey *)malloc(cap * sizeof(pairkey));
    for (size_t i = 0; i < cap; i++) s->e[i].km = EMPTY_KEY;
    s->capmask = cap - 1;
    s->n = 0;
}
static void pairset_free(pairset *s) { free(s->e); }
static inline size_t pairset_slot(const pairset *s, pairkey k) {
    return mix(k.km ^ mix(((uint64_t)k.a << 32) | k.b)) & s->capmask;
}
static int pairset_contains(const pairset *s, pairkey k) {
    size_t i = pairset_slot(s, k);
    while (s->e[i].km != EMPTY_KEY) {
        if (s->e[i].km == k.km && s->e[i].a == k.a && s->e[i].b == k.b) return 1;
        i = (i + 1) & s->capmask;
    }
    return 0;
}
static void pairset_insert(pairset *s, pairkey k) {
    if ((s->n + 1) * 2 > s->capmask + 1) {
        pairset o = *s;
        size_t cap = (o.capmask + 1) * 2;
        s->e = (pairkey *)malloc(cap * sizeof(pairkey));
        for (size_t i = 0; i < cap; i++) s->e[i].km = EMPTY_KEY;
        s->capmask = cap - 1;
        s->n = 0;
        for (size_t i = 0; i <= o.capmask; i++)
            if (o.e[i].km != EMPTY_KEY) pairset_insert(s, o.e[i]);
        free(o.e);
    }
    size_t i = pairset_slot(s, k);
    while (s->e[i].km != EMPTY_KEY) {
        if (s->e[i].km == k.km && s->e[i].a == k.a && s->e[i].b == k.b) return;
        i = (i + 1) & s->capmask;
    }
    s->e[i] = k;
    s->n++;
}

/* ------------------------------------------------------------------------------------------
 * L2: genome sketch
 * ---------------------------------------------------------------------------------------- */

typedef struct { uint64_t contig, pos, hash; } ctuple;
static int ctuple_cmp(const void *a, const void *b) {
    const ctuple *x = (const ctuple *)a, *y = (const ctuple *)b;
    if (x->contig != y->contig) return x->contig < y->contig ? -1 : 1;
    if (x->pos != y->pos) return x->pos < y->pos ? -1 : 1;
    if (x->hash != y->hash) return x->hash < y->hash ? -1 : 1;
    return 0;
}

/* src/sketch.rs:550-622 (sketch_genome); with individual semantics (:481-548) the caller passes
 * one contig at a time: contig_number is 0 and the `last_contig != contig` test never fires. */
int syo_sketch_genome(const uint8_t *bases, const uint64_t *contig_off, uint32_t n_contigs, int k,
                      uint64_t c, uint64_t min_spacing, int pseudotax, int sem,
                      uint64_t *out_kmers, size_t *n_kmers, uint64_t *out_tracked,
                      size_t *n_tracked, size_t cap, uint64_t *gn_size) {
    size_t total = 0, vcap = 1024;
    ctuple *vec = (ctuple *)malloc(vcap * sizeof(ctuple));
    uint64_t size = 0;
    for (uint32_t ci = 0; ci < n_contigs; ci++) {
        const uint8_t *s = bases + contig_off[ci];
        size_t len = (size_t)(contig_off[ci + 1] - contig_off[ci]);
        size += len; /* :581 — short contigs count too */
        size_t wcap = len >= (size_t)k ? len - (size_t)k + 1 : 0;
        size_t scap = wcap / 16 + 64;
        uint64_t *ph = NULL, *pp = NULL;
        size_t got;
        for (;;) {
            ph = (uint64_t *)malloc(scap * sizeof(uint64_t));
            pp = (uint64_t *)malloc(scap * sizeof(uint64_t));
            got = syo_extract_markers_positions(s, len, k, c, sem, pp, ph, scap);
            if (got == (size_t)-1) { free(ph); free(pp); free(vec); return 2; }
            if (got <= scap) break;
            free(ph); free(pp);
            scap = got;
        }
        if (total + got > vcap) {
            while (total + got > vcap) vcap *= 2;
            vec = (ctuple *)realloc(vec, vcap * sizeof(ctuple));
        }
        for (size_t i = 0; i < got; i++) {
            vec[total + i].contig = ci;
            vec[total + i].pos = pp[i];
            vec[total + i].hash = ph[i];
        }
        total += got;
        free(ph); free(pp);
    }
    *gn_size = size;
    qsort(vec, total, sizeof(ctuple), ctuple_cmp); /* :593 vec.sort() */
    /* :594-600 — a k-mer seen twice lands in duplicate_set */
    u64map seen;
    u64map_init(&seen, total);
    for (size_t i = 0; i < total; i++) {
        uint32_t *v = u64map_entry(&seen, vec[i].hash);
        if (*v < 2) (*v)++;
    }
    size_t nk = 0, nt = 0;
    int overflow = 0;
    uint64_t last_pos = 0, last_contig = 0;
    for (size_t i = 0; i < total; i++) { /* :602-614 */
        if (*u64map_find(&seen, vec[i].hash) >= 2) continue;
        if (last_pos == 0 || last_contig != vec[i].contig || vec[i].pos - last_pos > min_spacing) {
            if (nk < cap) out_kmers[nk] = vec[i].hash; else overflow = 1;
            nk++;
            last_contig = vec[i].contig;
            last_pos = vec[i].pos;
        } else if (pseudotax) {
            if (nt < cap) out_tracked[nt] = vec[i].hash; else overflow = 1;
            nt++;
        }
    }
    *n_kmers = nk;
    *n_tracked = nt;
    u64map_free(&seen);
    free(vec);
    return overflow;
}

/* ------------------------------------------------------------------------------------------
 * L2: read sketch (sample)
 * ---------------------------------------------------------------------------------------- */

/* src/sketch.rs:624-656 pair_kmer_single: Marker = u32 => 16 bases per key. */
static int pair_kmer_single(const uint8_t *s, size_t len, uint32_t p0[2], uint32_t p1[2]) {
    const size_t kk = 16;
    if (len < 4 * kk + 2) return 0;
    const uint8_t *L = lut();
    uint32_t f = 0, g = 0, r = 0, t = 0;
    size_t half = len / 2;
    for (size_t i = 0; i < kk; i++) {
        f = (f << 2) | L[s[2 * i]];
        r = (r << 2) | L[s[2 * i + half]];
        g = (g << 2) | L[s[1 + 2 * i]];
        t = (t << 2) | L[s[1 + 2 * i + half]];
    }
    p0[0] = f; p0[1] = r;
    p1[0] = g; p1[1] = t;
    return 1;
}

/* src/sketch.rs:690-731 dup_removal_lsh_full_exact; c_threshold = Some(MAX_DEDUP_COUNT=4) for single-end reads
 * (src/constants.rs:14, call :929-939), None = u32::MAX for read pairs with --fpr 0 (call :829-838). */
static void dup_removal_thr(u64map *counts, pairset *set, uint64_t km, int has_pair,
                            const uint32_t p0[2], const uint32_t p1[2], uint64_t *num_dup,
                            int no_dedup, uint32_t c_threshold) {
    uint32_t *c = u64map_entry(counts, km);
    if (!no_dedup && *c < c_threshold && has_pair) {
        int ret = 0;
        pairkey k0 = {km, p0[0], p0[1]}, k1 = {km, p1[0], p1[1]};
        if (pairset_contains(set, k0)) {
            if (*c > 0) ret = 1;
        } else {
            pairset_insert(set, k0);
        }
        if (pairset_contains(set, k1)) {
            if (*c > 0) ret = 1;
        } else {
            pairset_insert(set, k1);
        }
        if (ret) {
            (*num_dup)++;
            return;
        }
        /* pairset_insert may not move `counts`, so c stays valid */
    }
    (*c)++;
}

static void dup_removal(u64map *counts, pairset *set, uint64_t km, int has_pair,
                        const uint32_t p0[2], const uint32_t p1[2], uint64_t *num_dup,
                        int no_dedup) {
    dup_removal_thr(counts, set, km, has_pair, p0, p1, num_dup, no_dedup, 4u);
}

/* src/sketch.rs:658-688 pair_kmer: 16 bases at even / odd offsets from the START of each mate. */
static int pair_kmer(const uint8_t *s1, size_t len1, const uint8_t *s2, size_t len2, uint32_t p0[2], uint32_t p1[2]) {
    const size_t kk = 16;
    if (len1 < 2 * kk + 1 || len2 < 2 * kk + 1) return 0;
    const uint8_t *L = lut();
    uint32_t f = 0, g = 0, r = 0, t = 0;
    for (size_t i = 0; i < kk; i++) {
        f = (f << 2) | L[s1[2 * i]];
        r = (r << 2) | L[s2[2 * i]];
        g = (g << 2) | L[s1[1 + 2 * i]];
        t = (t << 2) | L[s2[1 + 2 * i]];
    }
    p0[0] = f; p0[1] = r;
    p1[0] = g; p1[1] = t;
    return 1;
}

typedef struct { uint64_t h; uint32_t c; } hc;
static int hc_cmp(const void *a, const void *b) {
    uint64_t x = ((const hc *)a)->h, y = ((const hc *)b)->h;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* src/sketch.rs:897-959 */
int syo_sketch_reads(const uint8_t *bases, const uint64_t *rec_off, uint64_t n_reads, int k,
                     uint64_t c, int no_dedup, int sem, int nthreads, uint64_t *out_hash,
                     uint32_t *out_count, size_t *n_out, size_t cap, double *mean_read_length,
                     uint64_t *num_dup_removed) {
    /* phase 1 (parallelisable): per-read survivor lists, kept in read order */
    int nchunks = nthreads > 1 ? nthreads * 8 : 1;
    if ((uint64_t)nchunks > n_reads) nchunks = n_reads ? (int)n_reads : 1;
    uint64_t **ch_hash = (uint64_t **)calloc((size_t)nchunks, sizeof(uint64_t *));
    uint32_t **ch_rel = (uint32_t **)calloc((size_t)nchunks, sizeof(uint32_t *)); /* read - chunk start */
    size_t *ch_n = (size_t *)calloc((size_t)nchunks, sizeof(size_t));
    int bad = 0;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads > 1 ? nthreads : 1)
#endif
    for (int ch = 0; ch < nchunks; ch++) {
        uint64_t r0 = n_reads * (uint64_t)ch / (uint64_t)nchunks;
        uint64_t r1 = n_reads * (uint64_t)(ch + 1) / (uint64_t)nchunks;
        uint64_t nb = rec_off[r1] - rec_off[r0];
        size_t vcap = (size_t)(nb / 64 + 1024), n = 0;
        uint64_t *vh = (uint64_t *)malloc(vcap * sizeof(uint64_t));
        uint32_t *vr = (uint32_t *)malloc(vcap * sizeof(uint32_t));
        for (uint64_t r = r0; r < r1; r++) {
            const uint8_t *s = bases + rec_off[r];
            size_t len = (size_t)(rec_off[r + 1] - rec_off[r]);
            size_t need = len >= (size_t)k ? len - (size_t)k + 1 : 0;
            if (n + need > vcap) {
                while (n + need > vcap) vcap *= 2;
                vh = (uint64_t *)realloc(vh, vcap * sizeof(uint64_t));
                vr = (uint32_t *)realloc(vr, vcap * sizeof(uint32_t));
            }
            size_t got = syo_extract_markers(s, len, k, c, sem, vh + n, vcap - n);
            if (got == (size_t)-1) { bad = 1; got = 0; }
            for (size_t i = 0; i < got; i++) vr[n + i] = (uint32_t)(r - r0);
            n += got;
        }
        ch_hash[ch] = vh; ch_rel[ch] = vr; ch_n[ch] = n;
    }
    if (bad) {
        for (int ch = 0; ch < nchunks; ch++) { free(ch_hash[ch]); free(ch_rel[ch]); }
        free(ch_hash); free(ch_rel); free(ch_n);
        return 2;
    }
    /* phase 2 (sequential, file order): the dedup state machine + running mean (:917-947) */
    size_t total = 0;
    for (int ch = 0; ch < nchunks; ch++) total += ch_n[ch];
    u64map counts;
    pairset set;
    u64map_init(&counts, total);
    pairset_init(&set, 1024);
    uint64_t ndup = 0;
    double mean = 0., counter = 0.;
    for (int ch = 0; ch < nchunks; ch++) {
        uint64_t r0 = n_reads * (uint64_t)ch / (uint64_t)nchunks;
        uint64_t r1 = n_reads * (uint64_t)(ch + 1) / (uint64_t)nchunks;
        size_t j = 0;
        for (uint64_t r = r0; r < r1; r++) {
            const uint8_t *s = bases + rec_off[r];
            size_t len = (size_t)(rec_off[r + 1] - rec_off[r]);
            uint32_t p0[2] = {0, 0}, p1[2] = {0, 0};
            int has_pair = 0;
            if (len <= 400) has_pair = pair_kmer_single(s, len, p0, p1); /* :923-927 */
            while (j < ch_n[ch] && ch_rel[ch][j] == (uint32_t)(r - r0)) {
                dup_removal(&counts, &set, ch_hash[ch][j], has_pair, p0, p1, &ndup, no_dedup);
                j++;
            }
            counter += 1.;
            mean = mean + (((double)len) - mean) / counter; /* :941-943 */
        }
        free(ch_hash[ch]); free(ch_rel[ch]);
    }
    free(ch_hash); free(ch_rel); free(ch_n);
    hc *arr = (hc *)malloc((counts.n + 1) * sizeof(hc));
    size_t n = 0;
    for (size_t i = 0; i <= counts.capmask; i++)
        if (counts.keys[i] != EMPTY_KEY) { arr[n].h = counts.keys[i]; arr[n].c = counts.vals[i]; n++; }
    qsort(arr, n, sizeof(hc), hc_cmp);
    int overflow = n > cap;
    for (size_t i = 0; i < n && i < cap; i++) { out_hash[i] = arr[i].h; out_count[i] = arr[i].c; }
    *n_out = n;
    if (mean_read_length) *mean_read_length = mean;
    if (num_dup_removed) *num_dup_removed = ndup;
    free(arr);
    u64map_free(&counts);
    pairset_free(&set);
    return overflow;
}

/* src/sketch.rs:771-895 sketch_pair_sequences with dedup_fpr == 0 (the exact set, :829-838 / :855-865; the
 * default approximate cuckoo filter is out of scope, SURVEY R11).  n_pairs = records zipped from the two
 * files.  Mate 1's k-mers first, then mate 2's that do not occur in mate 1 (:849-853). */
int syo_sketch_read_pairs(const uint8_t *bases1, const uint64_t *off1, const uint8_t *bases2, const uint64_t *off2,
                          uint64_t n_pairs, int k, uint64_t c, int no_dedup, int sem, uint64_t *out_hash,
                          uint32_t *out_count, size_t *n_out, size_t cap, double *mean_read_length,
                          uint64_t *num_dup_removed) {
    u64map counts;
    pairset set;
    u64map_init(&counts, 1024);
    pairset_init(&set, 1024);
    uint64_t ndup = 0;
    double mean = 0., counter = 0.;
    size_t vcap = 1024;
    uint64_t *v1 = (uint64_t *)malloc(vcap * sizeof(uint64_t)), *v2 = (uint64_t *)malloc(vcap * sizeof(uint64_t));
    for (uint64_t p = 0; p < n_pairs; p++) {
        const uint8_t *s1 = bases1 + off1[p], *s2 = bases2 + off2[p];
        const size_t l1 = (size_t)(off1[p + 1] - off1[p]), l2 = (size_t)(off2[p + 1] - off2[p]);
        const size_t need = (l1 > l2 ? l1 : l2) + 8;
        if (need > vcap) {
            vcap = need * 2;
            v1 = (uint64_t *)realloc(v1, vcap * sizeof(uint64_t));
            v2 = (uint64_t *)realloc(v2, vcap * sizeof(uint64_t));
        }
        const size_t n1 = syo_extract_markers(s1, l1, k, c, sem, v1, vcap);
        const size_t n2 = syo_extract_markers(s2, l2, k, c, sem, v2, vcap);
        if (n1 == (size_t)-1 || n2 == (size_t)-1) { free(v1); free(v2); u64map_free(&counts); pairset_free(&set); return 2; }
        uint32_t p0[2] = {0, 0}, p1[2] = {0, 0};
        const int has_pair = pair_kmer(s1, l1, s2, l2, p0, p1);
        counter += 1.;
        mean = mean + (((double)l1) - mean) / counter; /* :824-826 */
        for (size_t i = 0; i < n1; i++) dup_removal_thr(&counts, &set, v1[i], has_pair, p0, p1, &ndup, no_dedup, 0xFFFFFFFFu);
        for (size_t i = 0; i < n2; i++) {
            int in1 = 0;
            for (size_t j = 0; j < n1; j++) if (v1[j] == v2[i]) { in1 = 1; break; }   /* temp_vec1.contains(km) */
            if (in1) continue;
            dup_removal_thr(&counts, &set, v2[i], has_pair, p0, p1, &ndup, no_dedup, 0xFFFFFFFFu);
        }
    }
    free(v1); free(v2);
    hc *arr = (hc *)malloc((counts.n + 1) * sizeof(hc));
    size_t n = 0;
    for (size_t i = 0; i <= counts.capmask; i++)
        if (counts.keys[i] != EMPTY_KEY) { arr[n].h = counts.keys[i]; arr[n].c = counts.vals[i]; n++; }
    qsort(arr, n, sizeof(hc), hc_cmp);
    int overflow = n > cap;
    for (size_t i = 0; i < n && i < cap; i++) { out_hash[i] = arr[i].h; out_count[i] = arr[i].c; }
    *n_out = n;
    if (mean_read_length) *mean_read_length = mean;
    if (num_dup_removed) *num_dup_removed = ndup;
    free(arr);
    u64map_free(&counts);
    pairset_free(&set);
    return overflow;
}

/* ------------------------------------------------------------------------------------------
 * containment
 * ---------------------------------------------------------------------------------------- */

struct syo_sample { u64map m; };

syo_sample *syo_sample_new(const uint64_t *hash, const uint32_t *count, size_t n) {
    syo_sample *s = (syo_sample *)malloc(sizeof(syo_sample));
    u64map_init(&s->m, n);
    for (size_t i = 0; i < n; i++) *u64map_entry(&s->m, hash[i]) = count[i];
    return s;
}
void syo_sample_free(syo_sample *s) {
    if (!s) return;
    u64map_free(&s->m);
    free(s);
}

/* statrs 0.16.1 Poisson::cdf(x) = Q(x+1, lambda) = e^-lambda * sum_{i<=x} lambda^i/i! for
 * integer x; call site src/contain.rs:664,669. */
static double poisson_cdf(double lambda, uint64_t x) {
    long double term = expl(-(long double)lambda), sum = 0.0L;
    for (uint64_t i = 0; i <= x; i++) {
        sum += term;
        term *= (long double)lambda / (long double)(i + 1);
        if (i > 100000) break;
    }
    return (double)sum;
}

uint32_t syo_poisson_cutoff(uint32_t median) {
    uint32_t x = median, last = 0;
    for (;; x++) {
        if (poisson_cdf((double)median, x) < 0.9999999999) last = x; /* src/constants.rs:3 */
        else break;
    }
    return last;
}

static int u32_cmp(const void *a, const void *b) {
    uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* src/inference.rs:207-242. data need not be sorted. */
static int ratio_lambda(const uint32_t *full, size_t n, double min_count_correct, double *lam) {
    size_t num_zero = 0;
    uint32_t *nz = (uint32_t *)malloc((n + 1) * sizeof(uint32_t));
    size_t m = 0;
    for (size_t i = 0; i < n; i++) {
        if (full[i] == 0) num_zero++;
        else nz[m++] = full[i];
    }
    qsort(nz, m, sizeof(uint32_t), u32_cmp);
    /* run-length = count_map */
    size_t distinct = 0;
    uint32_t best_val = 0;
    size_t best_cnt = 0;
    for (size_t i = 0; i < m;) {
        size_t j = i;
        while (j < m && nz[j] == nz[i]) j++;
        distinct++;
        /* sort of (count,value) descending => max count, ties to the larger value (:226-230) */
        if (j - i > best_cnt || (j - i == best_cnt && nz[i] > best_val)) { best_cnt = j - i; best_val = nz[i]; }
        i = j;
    }
    int ok = 0;
    if (distinct == 1) goto done;               /* :221-223 */
    if (n - num_zero < 25) goto done;           /* SAMPLE_SIZE_CUTOFF, src/constants.rs:4 */
    {
        /* count of value best_val+1 */
        size_t cnt_p1 = 0;
        for (size_t i = 0; i < m; i++) if ((uint64_t)nz[i] == (uint64_t)best_val + 1) cnt_p1++;
        if (cnt_p1 == 0) goto done;             /* :231-233 */
        double count_p1 = (double)cnt_p1, count = (double)best_cnt;
        if (count_p1 < min_count_correct || count < min_count_correct) goto done;
        *lam = count_p1 / count * (double)((uint64_t)best_val + 1);
        ok = 1;
    }
done:
    free(nz);
    return ok;
}

/* The double nearest the 113-bit q; a q within 2^-100 (relative) of a midpoint between two doubles is counted in
 * *p->cr_undecided, since libquadmath's own error could then decide the rounding (tests/cpp/crmath_check.cpp
 * round_quad). */
static double cr_round(const syo_params *p, __float128 q) {
    const double y = (double)q;
    const double up = nextafter(y, INFINITY), dn = nextafter(y, 0.);
    const __float128 tol = fabsq(q) * (__float128)0x1p-100;
    if ((fabsq(q - ((__float128)y + (__float128)up) / 2) <= tol || fabsq(q - ((__float128)y + (__float128)dn) / 2) <= tol) &&
        p->cr_undecided)
        __atomic_fetch_add(p->cr_undecided, 1, __ATOMIC_RELAXED);
    return y;
}

/* the reference's ANI pow / exp: glibc, or correctly rounded under p->cr_math */
static double ani_pow(const syo_params *p, double x, double c) {
    return p->cr_math ? cr_round(p, powq((__float128)x, (__float128)c)) : pow(x, c);
}
static double ani_exp(const syo_params *p, double z) {
    return p->cr_math ? cr_round(p, expq((__float128)z)) : exp(z);
}

/* src/contain.rs:817-847 */
static int ani_from_lambda(const syo_params *p, int has_lambda, double lambda, double k, const uint32_t *full, size_t n,
                           double *ani_out) {
    if (!has_lambda) return 0;
    size_t contain = 0;
    for (size_t i = 0; i < n; i++) if (full[i] != 0) contain++;
    double adj = (double)contain / (1. - ani_exp(p, -lambda)) / (double)n;
    double ani = ani_pow(p, adj, 1. / k);
    if (ani < 0. || isnan(ani)) return 0;
    *ani_out = ani;
    return 1;
}

/* fastrand 2.1.1 (Cargo.lock:287): WyRand with the wyhash v4.2 constants; Rng::with_seed(s)
 * stores s verbatim; u64 output = lo ^ hi of (s+=C0) * (s ^ C1). */
typedef struct { uint64_t s; } wyrand;
static inline uint64_t wy_u64(wyrand *r) {
    r->s += 0x2d358dccaa6c78a5ull;
    __uint128_t t = (__uint128_t)r->s * (__uint128_t)(r->s ^ 0x8bb84b93962eacc9ull);
    return (uint64_t)t ^ (uint64_t)(t >> 64);
}
/* fastrand gen_mod_u64: Lemire's nearly-divisionless bounded draw. */
static inline uint64_t wy_mod(wyrand *r, uint64_t n) {
    uint64_t x = wy_u64(r);
    __uint128_t m = (__uint128_t)x * n;
    uint64_t hi = (uint64_t)(m >> 64), lo = (uint64_t)m;
    if (lo < n) {
        uint64_t t = (0 - n) % n;
        while (lo < t) {
            x = wy_u64(r);
            m = (__uint128_t)x * n;
            hi = (uint64_t)(m >> 64);
            lo = (uint64_t)m;
        }
    }
    return hi;
}

uint64_t syo_fastrand_usize(uint64_t seed, uint64_t n_draw, uint64_t range) {
    wyrand r = {seed};
    uint64_t v = 0;
    for (uint64_t i = 0; i < n_draw; i++) v = wy_mod(&r, range);
    return v;
}

static int dbl_cmp(const void *a, const void *b) {
    double x = *(const double *)a, y = *(const double *)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* src/contain.rs:849-898 */
static int bootstrap_interval(const syo_params *p, const uint32_t *full, size_t n, double k, double min_count_correct,
                              double ci[4]) {
    wyrand rng = {7}; /* fastrand::seed(7) :854 */
    const int iters = 100;
    double res_ani[100], res_lambda[100];
    int suc = 0;
    uint32_t *rv = (uint32_t *)malloc((n + 1) * sizeof(uint32_t));
    for (int it = 0; it < iters; it++) {
        for (size_t j = 0; j < n; j++) rv[j] = full[wy_mod(&rng, (uint64_t)n)];
        double lam = 0., ani = 0.;
        int hl = ratio_lambda(rv, n, min_count_correct, &lam);
        int ha = ani_from_lambda(p, hl, lam, k, rv, n, &ani);
        if (ha && hl && !isnan(ani) && !isnan(lam)) {
            res_ani[suc] = ani;
            res_lambda[suc] = lam;
            suc++;
        }
    }
    free(rv);
    if (suc < 50) return 0;
    qsort(res_ani, (size_t)suc, sizeof(double), dbl_cmp);
    qsort(res_lambda, (size_t)suc, sizeof(double), dbl_cmp);
    ci[0] = res_ani[suc * 5 / 100 - 1];
    ci[1] = res_ani[suc * 95 / 100 - 1];
    ci[2] = res_lambda[suc * 5 / 100 - 1];
    ci[3] = res_lambda[suc * 95 / 100 - 1];
    return 1;
}

/* winner map: kmer -> (ani, genome) (src/contain.rs:410-430) */
typedef struct {
    uint64_t *keys;
    double *ani;
    uint32_t *gen;
    size_t capmask, n;
} winmap;
static void winmap_init(winmap *m, size_t expect) {
    size_t cap = 16;
    while (cap < expect * 2 + 2) cap <<= 1;
    m->keys = (uint64_t *)malloc(cap * sizeof(uint64_t));
    m->ani = (double *)malloc(cap * sizeof(double));
    m->gen = (uint32_t *)malloc(cap * sizeof(uint32_t));
    for (size_t i = 0; i < cap; i++) m->keys[i] = EMPTY_KEY;
    m->capmask = cap - 1;
    m->n = 0;
}
static void winmap_free(winmap *m) { free(m->keys); free(m->ani); free(m->gen); }
static void winmap_offer(winmap *m, uint64_t key, double ani, uint32_t gen) {
    size_t i = mix(key) & m->capmask;
    while (m->keys[i] != EMPTY_KEY) {
        if (m->keys[i] == key) {
            if (ani > m->ani[i]) { m->ani[i] = ani; m->gen[i] = gen; } /* strict > : first wins ties */
            return;
        }
        i = (i + 1) & m->capmask;
    }
    m->keys[i] = key; m->ani[i] = ani; m->gen[i] = gen; m->n++;
}
static uint32_t winmap_get(const winmap *m, uint64_t key) {
    size_t i = mix(key) & m->capmask;
    while (m->keys[i] != EMPTY_KEY) {
        if (m->keys[i] == key) return m->gen[i];
        i = (i + 1) & m->capmask;
    }
    return UINT32_MAX;
}

/* src/contain.rs:601-814 */
static int get_stats(const syo_params *p, const uint64_t *gk, size_t n, const syo_sample *sample,
                     const winmap *winner, uint32_t genome_index, syo_ani_result *out) {
    if ((double)n < p->min_number_kmers) return 0; /* :627 */
    size_t contain = 0, lost = 0;
    uint32_t *covs = (uint32_t *)malloc((n + 1) * sizeof(uint32_t));
    for (size_t i = 0; i < n; i++) { /* :632-652 */
        const uint32_t *c = u64map_find(&sample->m, gk[i]);
        if (!c) continue;
        if (*c == 0) continue;
        if (winner) {
            if (winmap_get(winner, gk[i]) != genome_index) { lost++; continue; }
        }
        covs[contain++] = *c;
    }
    if (contain == 0) { free(covs); return 0; } /* :654 */
    double k = (double)p->k;
    double naive_ani = ani_pow(p, (double)contain / (double)n, 1. / k);
    qsort(covs, contain, sizeof(uint32_t), u32_cmp);
    double median = (double)covs[contain / 2];
    double max_cov = 1.7976931348623157e308; /* f64::MAX */
    if (median < 30.) { /* :664-675 */
        for (size_t i = contain / 2; i < contain; i++) {
            if (poisson_cdf(median, covs[i]) < 0.9999999999) max_cov = (double)covs[i];
            else break;
        }
    }
    size_t nfull = n - contain;
    uint32_t *full = (uint32_t *)calloc(n + 1, sizeof(uint32_t));
    for (size_t i = 0; i < contain; i++)
        if ((double)covs[i] <= max_cov) full[nfull++] = covs[i];
    uint32_t sum = 0; /* iter().sum::<u32>() — wraps in release builds */
    for (size_t i = 0; i < nfull; i++) sum += full[i];
    double mean_cov = (double)sum / (double)nfull;
    double geq1_mean = (double)sum / (double)contain; /* :690 */
    (void)mean_cov;
    uint32_t status;
    double lam = 0.;
    if (median > 2.) status = SYO_LAMBDA_HIGH; /* MEDIAN_ANI_THRESHOLD */
    else status = ratio_lambda(full, nfull, p->min_count_correct, &lam) ? SYO_LAMBDA_VALUE : SYO_LAMBDA_LOW;
    double final_cov;
    if (status == SYO_LAMBDA_VALUE) final_cov = lam;
    else if (median < 15.) final_cov = geq1_mean; /* MAX_MEDIAN_FOR_MEAN_FINAL_EST */
    else final_cov = p->mean_coverage ? geq1_mean : median;
    int has_lambda = status == SYO_LAMBDA_VALUE;
    double est_ani = 0.;
    int has_est = ani_from_lambda(p, has_lambda, final_cov, k, full, nfull, &est_ani);
    double final_ani = (!has_lambda || !has_est || p->no_adj) ? naive_ani : est_ani;
    double min_ani = p->minimum_ani >= 0. ? p->minimum_ani / 100. : (p->pseudotax ? 0.95 : 0.90);
    if (final_ani < min_ani) { free(covs); free(full); return 0; }
    memset(out, 0, sizeof(*out));
    if (!p->no_ci && has_lambda)
        out->ci_valid = (uint32_t)bootstrap_interval(p, full, nfull, k, p->min_count_correct, out->ci);
    out->genome = genome_index;
    out->lambda_status = status;
    out->contain = contain;
    out->glen = n;
    out->kmers_lost = winner ? (int64_t)lost : -1;
    out->naive_ani = naive_ani;
    out->final_est_ani = final_ani;
    out->final_est_cov = final_cov;
    out->mean_cov = geq1_mean;
    out->median_cov = median;
    out->lambda = has_lambda ? lam : 0.;
    free(covs);
    free(full);
    return 1;
}

int syo_get_stats(const syo_params *p, const uint64_t *genome_kmers, size_t n,
                  const syo_sample *sample, uint32_t genome_index, syo_ani_result *out) {
    return get_stats(p, genome_kmers, n, sample, NULL, genome_index, out);
}

typedef struct { double key; size_t idx; } sortkey;
static int sortkey_desc(const void *a, const void *b) {
    const sortkey *x = (const sortkey *)a, *y = (const sortkey *)b;
    if (x->key > y->key) return -1;
    if (x->key < y->key) return 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx ? 1 : 0); /* stable */
}

/* -u / --estimate-unknown with an explicit --read-seq-id (src/contain.rs:274-279: kmer_id = (seq_id/100)^k; the
 * automatic estimate get_kmer_identity :901-951 walks the hash map in iteration order and is out of scope):
 * estimate_true_cov (:377-389) and estimate_covered_bases (:391-408). */
static void estimate_true_cov(syo_ani_result *res, size_t n, double kmer_id, double read_length, int k) {
    const double multiplier = read_length / (read_length - (double)k + 1.);
    for (size_t i = 0; i < n; i++) res[i].final_est_cov = res[i].final_est_cov / kmer_id * multiplier;
}

static int64_t contain_sample_impl(const syo_params *p, const uint64_t *kmers, const uint64_t *kmer_off,
                                   const uint64_t *tracked, const uint64_t *tracked_off,
                                   const uint64_t *gn_size, uint32_t n_genomes, const syo_sample *sample,
                                   int nthreads, syo_ani_result *out, size_t cap, const syo_unknown *u);

int64_t syo_contain_sample(const syo_params *p, const uint64_t *kmers, const uint64_t *kmer_off,
                           const uint64_t *tracked, const uint64_t *tracked_off,
                           const uint64_t *gn_size, uint32_t n_genomes, const syo_sample *sample,
                           int nthreads, syo_ani_result *out, size_t cap) {
    return contain_sample_impl(p, kmers, kmer_off, tracked, tracked_off, gn_size, n_genomes, sample, nthreads, out, cap, NULL);
}

int64_t syo_contain_sample_unknown(const syo_params *p, const uint64_t *kmers, const uint64_t *kmer_off,
                                   const uint64_t *tracked, const uint64_t *tracked_off,
                                   const uint64_t *gn_size, uint32_t n_genomes, const syo_sample *sample,
                                   int nthreads, syo_ani_result *out, size_t cap, const syo_unknown *u) {
    return contain_sample_impl(p, kmers, kmer_off, tracked, tracked_off, gn_size, n_genomes, sample, nthreads, out, cap, u);
}

static int64_t contain_sample_impl(const syo_params *p, const uint64_t *kmers, const uint64_t *kmer_off,
                                   const uint64_t *tracked, const uint64_t *tracked_off,
                                   const uint64_t *gn_size, uint32_t n_genomes, const syo_sample *sample,
                                   int nthreads, syo_ani_result *out, size_t cap, const syo_unknown *u) {
    const double kmer_id = u ? pow(u->read_seq_id / 100., (double)p->k) : 1.;
    /* pass 1 (:284-292): par_iter over genomes */
    syo_ani_result *r1 = (syo_ani_result *)malloc(((size_t)n_genomes + 1) * sizeof(syo_ani_result));
    uint8_t *ok1 = (uint8_t *)calloc((size_t)n_genomes + 1, 1);
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthreads > 1 ? nthreads : 1)
#endif
    for (int64_t g = 0; g < (int64_t)n_genomes; g++)
        ok1[g] = (uint8_t)get_stats(p, kmers + kmer_off[g], (size_t)(kmer_off[g + 1] - kmer_off[g]),
                                    sample, NULL, (uint32_t)g, &r1[g]);
    size_t n1 = 0;
    for (uint32_t g = 0; g < n_genomes; g++)
        if (ok1[g]) r1[n1++] = r1[g]; /* compact, genome-index order */
    syo_ani_result *res = r1;
    size_t nres = n1;
    syo_ani_result *r2 = NULL;
    if (u) estimate_true_cov(r1, n1, kmer_id, u->mean_read_length, p->k); /* :295 */
    if (p->pseudotax) {
        /* winner_table (:410-430) */
        size_t tot = 0;
        for (size_t i = 0; i < n1; i++) {
            uint32_t g = r1[i].genome;
            tot += (size_t)(kmer_off[g + 1] - kmer_off[g]);
            if (tracked_off) tot += (size_t)(tracked_off[g + 1] - tracked_off[g]);
        }
        winmap w;
        winmap_init(&w, tot);
        for (size_t i = 0; i < n1; i++) {
            uint32_t g = r1[i].genome;
            for (uint64_t j = kmer_off[g]; j < kmer_off[g + 1]; j++)
                winmap_offer(&w, kmers[j], r1[i].final_est_ani, g);
            if (tracked_off)
                for (uint64_t j = tracked_off[g]; j < tracked_off[g + 1]; j++)
                    winmap_offer(&w, tracked[j], r1[i].final_est_ani, g);
        }
        /* pass 2 (:302-307) + derep_if_reassign_threshold (:353-375) */
        r2 = (syo_ani_result *)malloc((n1 + 1) * sizeof(syo_ani_result));
        uint8_t *ok2 = (uint8_t *)calloc(n1 + 1, 1);
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4) num_threads(nthreads > 1 ? nthreads : 1)
#endif
        for (int64_t i = 0; i < (int64_t)n1; i++) {
            uint32_t g = r1[i].genome;
            ok2[i] = (uint8_t)get_stats(p, kmers + kmer_off[g], (size_t)(kmer_off[g + 1] - kmer_off[g]),
                                        sample, &w, g, &r2[i]);
        }
        double threshold = pow(p->redundant_ani / 100., (double)p->k);
        size_t n2 = 0;
        for (size_t i = 0; i < n1; i++) {
            if (!ok2[i]) continue;
            double num_reassign = (double)(r1[i].contain - r2[i].contain);
            double reass_thresh = threshold * (double)r2[i].glen;
            if (num_reassign < reass_thresh) r2[n2++] = r2[i];
        }
        free(ok2);
        winmap_free(&w);
        double bases_explained = 1.;
        if (u) {
            estimate_true_cov(r2, n2, kmer_id, u->mean_read_length, p->k); /* :310 */
            /* estimate_covered_bases :391-408 */
            const double multiplier = u->mean_read_length / (u->mean_read_length - (double)p->k + 1.);
            double covered = 0.;
            for (size_t i = 0; i < n2; i++) covered += (double)gn_size[r2[i].genome] * r2[i].final_est_cov;
            uint64_t total_counts = 0;
            for (size_t i = 0; i <= sample->m.capmask; i++)
                if (sample->m.keys[i] != EMPTY_KEY) total_counts += sample->m.vals[i];
            const double tentative = (double)(u->sample_c * total_counts) * multiplier;
            bases_explained = tentative == 0. ? 0. : (covered / tentative < 1. ? covered / tentative : 1.);
        }
        /* abundances (:319-326) */
        double total_cov = 0., total_seq_cov = 0.;
        for (size_t i = 0; i < n2; i++) {
            total_cov += r2[i].final_est_cov;
            total_seq_cov += r2[i].final_est_cov * (double)gn_size[r2[i].genome];
        }
        for (size_t i = 0; i < n2; i++) {
            r2[i].rel_abund = r2[i].final_est_cov / total_cov * 100.;
            r2[i].seq_abund = r2[i].final_est_cov * (double)gn_size[r2[i].genome] / total_seq_cov * 100. * bases_explained;
        }
        res = r2;
        nres = n2;
    }
    /* sort (:329-334), stable */
    sortkey *sk = (sortkey *)malloc((nres + 1) * sizeof(sortkey));
    for (size_t i = 0; i < nres; i++) {
        sk[i].key = p->pseudotax ? res[i].rel_abund : res[i].final_est_ani;
        sk[i].idx = i;
    }
    qsort(sk, nres, sizeof(sortkey), sortkey_desc);
    int64_t ret = (int64_t)nres;
    if (nres > cap) ret = -1;
    else for (size_t i = 0; i < nres; i++) out[i] = res[sk[i].idx];
    free(sk);
    free(r1);
    free(r2);
    free(ok1);
    return ret;
}

/* src/contain.rs:18-94 */
int syo_format_row(const syo_ani_result *r, int pseudotax, const char *seq_name,
                   const char *gn_name, const char *contig_name, char *buf, size_t buflen) {
    char final_ani[64], lambda_print[64], ci_ani[96], ci_lambda[96];
    double fa = r->final_est_ani * 100.;
    snprintf(final_ani, sizeof final_ani, "%.2f", fa < 100. ? fa : 100.);
    if (r->lambda_status == SYO_LAMBDA_VALUE) snprintf(lambda_print, sizeof lambda_print, "%.3f", r->lambda);
    else if (r->lambda_status == SYO_LAMBDA_HIGH) snprintf(lambda_print, sizeof lambda_print, "HIGH");
    else snprintf(lambda_print, sizeof lambda_print, "LOW");
    if (!r->ci_valid) {
        snprintf(ci_ani, sizeof ci_ani, "NA-NA");
        snprintf(ci_lambda, sizeof ci_lambda, "NA-NA");
    } else {
        snprintf(ci_ani, sizeof ci_ani, "%.2f-%.2f", r->ci[0] * 100., r->ci[1] * 100.);
        snprintf(ci_lambda, sizeof ci_lambda, "%.2f-%.2f", r->ci[2], r->ci[3]);
    }
    int n;
    if (!pseudotax) {
        n = snprintf(buf, buflen, "%s\t%s\t%s\t%.3f\t%s\t%s\t%s\t%.0f\t%.3f\t%llu/%llu\t%.2f\t%s",
                     seq_name, gn_name, final_ani, r->final_est_cov, ci_ani, lambda_print, ci_lambda,
                     r->median_cov, r->mean_cov, (unsigned long long)r->contain,
                     (unsigned long long)r->glen, r->naive_ani * 100., contig_name);
    } else {
        n = snprintf(buf, buflen,
                     "%s\t%s\t%.4f\t%.4f\t%s\t%.3f\t%s\t%s\t%s\t%.0f\t%.3f\t%llu/%llu\t%.2f\t%lld\t%s",
                     seq_name, gn_name, r->rel_abund, r->seq_abund, final_ani, r->final_est_cov, ci_ani,
                     lambda_print, ci_lambda, r->median_cov, r->mean_cov,
                     (unsigned long long)r->contain, (unsigned long long)r->glen, r->naive_ani * 100.,
                     (long long)r->kmers_lost, contig_name);
    }
    return n;
}
