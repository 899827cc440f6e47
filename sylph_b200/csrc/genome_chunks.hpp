// genome_chunks.hpp — how a host-memory genome batch is cut into chunks for the host feeder (ingest.hpp).  Host-only and
// free of CUDA, so that tests/cpp/genome_chunks_check.cpp can build it with a plain C++ compiler.
#pragma once

#include <cstdint>
#include <vector>

namespace syl {

// Genomes [g0, g1) = contigs [c0, c1) = bases [contig_off[c0], contig_off[c1]).  own: the chunk exceeds a cap (it is one
// genome larger than a chunk) and goes through a device buffer of its own instead of a ring slot.
struct GenomeChunk {
    uint64_t g0, g1, c0, c1;
    bool own;
};

// Cut genomes [0, n_genomes) into chunks of whole genomes, greedily in genome order: a chunk holds at most max_bases
// bases and max_contigs contigs, unless its one genome alone exceeds them.  genome_off == NULL: every contig is a genome
// (n_genomes contigs).  The genome post-pass needs all survivors of a genome at once, so no genome is ever split.
// Genomes without contigs or bases join the chunk in front of them, or start the next one after an own chunk.
inline void plan_genome_chunks(const uint64_t *contig_off, const uint64_t *genome_off, uint64_t n_genomes,
                               uint64_t max_bases, uint64_t max_contigs, std::vector<GenomeChunk> &chunks) {
    auto first_contig = [&](uint64_t g) { return genome_off ? genome_off[g] : g; };
    uint64_t g = 0;
    while (g < n_genomes) {
        const uint64_t c0 = first_contig(g), b0 = contig_off[c0];
        uint64_t g1 = g + 1;
        const bool own = contig_off[first_contig(g1)] - b0 > max_bases || first_contig(g1) - c0 > max_contigs;
        if (!own)
            while (g1 < n_genomes && contig_off[first_contig(g1 + 1)] - b0 <= max_bases && first_contig(g1 + 1) - c0 <= max_contigs) g1++;
        chunks.push_back({g, g1, c0, first_contig(g1), own});
        g = g1;
    }
}

}  // namespace syl
