// Host build of sample_batches.hpp (the rule syl_query_host_samples / syl_profile_host_samples cut samples by).
//
// stdin, one case per line: "S G budget max_pairs max_kmers max_samples per_kmer per_sample per_hit per_pair fixed
// off[0..S]".  stdout, one line per case: "ok first[0] first[1] ...", "oom <sample> <bytes>" or "kmers <sample> <n>".
#include <cstdint>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "sample_batches.hpp"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        uint64_t S = 0, G = 0, budget = 0, max_pairs = 0, max_kmers = 0, max_samples = 0;
        syl::BatchCost c{};
        in >> S >> G >> budget >> max_pairs >> max_kmers >> max_samples >> c.per_kmer >> c.per_sample >> c.per_hit >> c.per_pair >> c.fixed;
        std::vector<uint64_t> off(S + 1);
        for (uint64_t &v : off) in >> v;
        std::vector<uint32_t> first;
        uint32_t bad = 0;
        uint64_t need = 0;
        switch (syl::plan_sample_batches(off.data(), (uint32_t)S, G, budget, max_pairs, max_kmers, (uint32_t)max_samples, c, first,
                                         &bad, &need)) {
            case syl::BATCH_OK:
                std::cout << "ok";
                for (uint32_t f : first) std::cout << " " << f;
                std::cout << "\n";
                break;
            case syl::BATCH_OOM: std::cout << "oom " << bad << " " << need << "\n"; break;
            default: std::cout << "kmers " << bad << " " << need << "\n"; break;
        }
    }
    return 0;
}
