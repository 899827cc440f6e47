// scan_plan.hpp — when a query or profile call on a host-memory database (syl_db_shards) streams the genome k-mers past
// the samples' lookup tables instead of building an index, how the database is cut into scan chunks, and the layout of
// a sample's lookup table.  Host-only and free of CUDA (the table helpers also compile for the device), so that
// tests/cpp/scan_plan_check.cpp can build it with a plain C++ compiler.
#pragma once

#include <cstdint>
#include <vector>

#include "shard_cut.hpp"

#ifdef __CUDACC__
#define SYL_HD __host__ __device__ __forceinline__
#else
#define SYL_HD inline
#endif

namespace syl {

// ---- the rule ------------------------------------------------------------------------------------------------------
// Costs of one call measured by scripts/time_db_scan.py (DESIGN.md §10) on an H100 80GB HBM3 at 700 W, on databases of
// 1.7e8, 2.9e8 and 6.0e8 index entries (85 % genome k-mers), samples of 64 genomes (about 1.1e6 k-mers each), in ns:
//   build   per index entry: 4.0 from pageable host arrays (6.0e8: 2.2-2.7 s), 0.8 from pinned ones (0.39-0.70 s); the
//           joins on the built index take milliseconds;
//   scan    the larger of the link and the probes, which overlap.  Link per genome k-mer: 1.3 pageable (through the
//           pinned ring; 6.0e8: 0.7 s), 0.2 pinned (0.1 s).  Probes per genome k-mer and sample: 0.02 while all
//           samples' tables fit the 50 MB L2 (k_scan at 1 and 4 samples: 0.020-0.022), 0.07 once they do not (k_scan at
//           64 samples 0.060, plus 0.01 of per-chunk statistics and rows seen in the wall time).  64 samples from
//           pageable arrays sit at the crossover: query even, profile's build ahead by 0.2-0.4 s at 2.9e8 entries.
constexpr double BUILD_NS_PAGEABLE = 4.0, BUILD_NS_PINNED = 0.8;
constexpr double LINK_NS_PAGEABLE = 1.3, LINK_NS_PINNED = 0.2;
constexpr double PROBE_NS_IN_L2 = 0.02, PROBE_NS_BEYOND_L2 = 0.07;
// What a probe that misses touches per sample key (almost every genome k-mer misses): its fingerprint (4 bytes) and
// directory (about 2).  Samples of 1.1e6 keys: 4 fit the 50 MB L2 together (measured 0.021 ns), 16 do not (0.043).
constexpr double TABLE_BYTES_PER_KEY = 6;
constexpr double L2_BYTES = 50e6;
// Below this many index entries a call never scans, whatever the model says: small databases keep the index path,
// whose build takes about a second there (pageable arrays).  The floor is a policy, not a crossover: DESIGN.md §10
// measures the scan ahead of the build for few samples at 1.7e8 entries (below it) and 2.9e8 (just above) as well.
constexpr uint64_t SCAN_MIN_ENTRIES = 1ull << 28;

struct ScanShape {
    uint64_t n_kmers, n_tracked, n_genomes;
    uint32_t n_samples;
    uint64_t sample_kmers;  // all samples' k-mers together
    bool one_batch;         // the samples fit one sample batch (a scan keeps them all on the device at once)
    bool pinned;            // the genome k-mers are in pinned host memory
};

// true: scan; false: build the index shard by shard
inline bool scan_wins(const ScanShape &s) {
    if (!s.one_batch || s.n_samples == 0 || s.n_genomes == 0) return false;
    const double entries = (double)(s.n_kmers + s.n_tracked), nk = (double)s.n_kmers;
    if (s.n_kmers + s.n_tracked < SCAN_MIN_ENTRIES) return false;
    const double probe = TABLE_BYTES_PER_KEY * (double)s.sample_kmers <= L2_BYTES ? PROBE_NS_IN_L2 : PROBE_NS_BEYOND_L2;
    const double link = (s.pinned ? LINK_NS_PINNED : LINK_NS_PAGEABLE) * nk, probes = probe * (double)s.n_samples * nk;
    const double build = (s.pinned ? BUILD_NS_PINNED : BUILD_NS_PAGEABLE) * entries;
    return (link > probes ? link : probes) < build;
}

// SYL_DB_SCAN forces either path ("0": build, "1": scan); anything else, or unset, leaves it to scan_wins.  Read per call.
inline int scan_forced(const char *env) {
    if (env && env[0] == '0' && !env[1]) return 0;
    if (env && env[0] == '1' && !env[1]) return 1;
    return -1;
}

// The decision of a call (forced: scan_forced's value).  A scan keeps all samples of the call on the device in one
// batch, so samples that do not fit one batch are never scanned, forced or not.
inline bool scan_decision(const ScanShape &s, int forced) {
    if (!s.one_batch || s.n_samples == 0 || s.n_genomes == 0) return false;
    return forced >= 0 ? forced == 1 : scan_wins(s);
}

// ---- the chunks ----------------------------------------------------------------------------------------------------
constexpr uint64_t SCAN_CHUNK = 1ull << 25;  // genome k-mers per scan chunk (SYL_DB_SCAN_CHUNK overrides it)

// Cut genomes [0, G) into scan chunks of whole genomes: at most `entries` genome k-mers (tracked k-mers never cross the
// link) and `genomes` genomes each, greedily in genome order; a genome larger than a chunk is a chunk of its own, and
// empty genomes join the chunk in front of them (or start the next one after a chunk over the cap).  chunk i = genomes [first[i], first[i + 1]).
inline void cut_scan_chunks(const uint64_t *kmer_off, uint64_t G, uint64_t entries, uint64_t genomes, std::vector<uint64_t> &first) {
    uint64_t bad = 0;
    cut_shards(kmer_off, nullptr, G, entries ? entries : 1, first, &bad, genomes ? genomes : 1);
}

// ---- a sample's lookup table ---------------------------------------------------------------------------------------
// Over the sample's hashes sorted ascending (n keys): NB = max(n / 2, 1) buckets, bucket(key) = mulhi(key, M) clamped
// to NB - 1 with M = NB * 2^64 / (maxkey + 1), as the index directory (contain.hpp bucket_of).  dir[b] = index of the
// first key whose bucket is >= b, for b = 0 .. NB (dir[NB] = n), and fp[i] = the low 32 bits of key i.  A probe reads
// dir[b], dir[b + 1] and the fingerprints between them; only a fingerprint match reads the key and its count.  Bytes
// beyond the sample itself: 4 per key (fp) and about 2 per key (dir).
SYL_HD uint64_t table_buckets(uint64_t n) { return n / 2 > 1 ? n / 2 : 1; }

SYL_HD uint64_t table_mult(uint64_t maxkey, uint64_t NB) {
    const unsigned __int128 m = ((unsigned __int128)NB << 64) / ((unsigned __int128)maxkey + 1);
    return m > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)m;
}

SYL_HD uint64_t table_bucket(uint64_t key, uint64_t M, uint64_t NB) {
    const uint64_t b = (uint64_t)(((unsigned __int128)key * M) >> 64);
    return b < NB ? b : NB - 1;
}

// the directory entries key i of the sorted keys[0 .. n) writes: those between its predecessor's bucket and its own
// (and, for the last key, those after its bucket, which hold n).  Every i of 0 .. n - 1 together write dir[0 .. NB];
// an empty sample has dir = {0, 0}.
SYL_HD void table_dir_entries(const uint64_t *keys, uint64_t n, uint64_t i, uint64_t M, uint64_t NB, uint32_t *dir) {
    const uint64_t b = table_bucket(keys[i], M, NB);
    const uint64_t from = i ? table_bucket(keys[i - 1], M, NB) + 1 : 0;
    for (uint64_t x = from; x <= b; x++) dir[x] = (uint32_t)i;
    if (i + 1 == n)
        for (uint64_t x = b + 1; x <= NB; x++) dir[x] = (uint32_t)n;
}

}  // namespace syl
