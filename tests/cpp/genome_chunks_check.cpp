// Host build of genome_chunks.hpp (how a host-memory genome batch is cut into chunks of whole genomes).
//
// stdin, one case per line: "max_bases max_contigs individual n_contigs contig_off[0..n_contigs] n_genomes
// genome_off[0..n_genomes]" (individual != 0: no genome offsets follow n_genomes, every contig is a genome).
// stdout, per case: "P" followed by P lines "g0 g1 c0 c1 own".
#include <cstdint>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "genome_chunks.hpp"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        uint64_t max_bases = 0, max_contigs = 0, n_contigs = 0, n_genomes = 0;
        int individual = 0;
        in >> max_bases >> max_contigs >> individual >> n_contigs;
        std::vector<uint64_t> contig_off(n_contigs + 1), genome_off;
        for (uint64_t &x : contig_off) in >> x;
        in >> n_genomes;
        if (!individual) {
            genome_off.resize(n_genomes + 1);
            for (uint64_t &x : genome_off) in >> x;
        }
        std::vector<syl::GenomeChunk> chunks;
        syl::plan_genome_chunks(contig_off.data(), individual ? nullptr : genome_off.data(), n_genomes, max_bases, max_contigs, chunks);
        std::cout << chunks.size() << "\n";
        for (const syl::GenomeChunk &c : chunks)
            std::cout << c.g0 << " " << c.g1 << " " << c.c0 << " " << c.c1 << " " << (c.own ? 1 : 0) << "\n";
    }
    return 0;
}
