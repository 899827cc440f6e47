// shard_cut.hpp — how syl_db_shards_create cuts a database into index shards.  Host-only and free of CUDA, so that
// tests/cpp/shard_cut_check.cpp can build it with a plain C++ compiler.
#pragma once

#include <cstdint>
#include <vector>

namespace syl {

constexpr uint64_t SHARD_MAX_ENTRIES = 0xFFFFFFFDull;  // 2^32 - 3: the largest index (k-mers + tracked) of one syl_db
constexpr uint64_t SHARD_MAX_GENOMES = 0x7FFFFFFEull;  // 2^31 - 2: the most genomes of one syl_db

// Index entries of genome g: its k-mers plus its tracked k-mers (tracked_off may be NULL).
inline uint64_t genome_entries(const uint64_t *kmer_off, const uint64_t *tracked_off, uint64_t g) {
    return kmer_off[g + 1] - kmer_off[g] + (tracked_off ? tracked_off[g + 1] - tracked_off[g] : 0);
}

// Cut genomes [0, G) into contiguous shards, greedily in genome order: shard i is [first[i], first[i + 1]), holds at most
// `cap` entries (capped at SHARD_MAX_ENTRIES) and `max_genomes` genomes.  A genome with more than `cap` entries is a
// shard of its own.  Offsets must be monotone.  Returns false, with *bad = the genome, when a genome alone holds more
// than SHARD_MAX_ENTRIES entries.  G == 0 gives no shard (first = {0}).
inline bool cut_shards(const uint64_t *kmer_off, const uint64_t *tracked_off, uint64_t G, uint64_t cap,
                       std::vector<uint64_t> &first, uint64_t *bad, uint64_t max_genomes = SHARD_MAX_GENOMES) {
    if (cap == 0 || cap > SHARD_MAX_ENTRIES) cap = SHARD_MAX_ENTRIES;
    first.assign(1, 0);
    uint64_t n = 0, g0 = 0;
    for (uint64_t g = 0; g < G; g++) {
        const uint64_t e = genome_entries(kmer_off, tracked_off, g);
        if (e > SHARD_MAX_ENTRIES) {
            *bad = g;
            return false;
        }
        if (g > g0 && (n + e > cap || g - g0 >= max_genomes)) {
            first.push_back(g);
            g0 = g;
            n = 0;
        }
        n += e;
    }
    if (G) first.push_back(G);
    return true;
}

}  // namespace syl
