// Host build of shard_cut.hpp (the rule syl_db_shards_create cuts a database by).
//
// stdin, one case per line: "G cap kmer_off[0..G] tracked_off[0..G]" with "-" in place of tracked_off for a database
// without tracked k-mers.  stdout, one line per case: "ok first[0] first[1] ..." or "bad <genome>".
#include <cstdint>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "shard_cut.hpp"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        uint64_t G = 0, cap = 0;
        in >> G >> cap;
        std::vector<uint64_t> ko(G + 1), to;
        for (uint64_t &v : ko) in >> v;
        std::string t;
        in >> t;
        if (t != "-") {
            to.resize(G + 1);
            to[0] = std::stoull(t);
            for (uint64_t i = 1; i <= G; i++) in >> to[i];
        }
        std::vector<uint64_t> first;
        uint64_t bad = 0;
        if (!syl::cut_shards(ko.data(), to.empty() ? nullptr : to.data(), G, cap, first, &bad)) {
            std::cout << "bad " << bad << "\n";
            continue;
        }
        std::cout << "ok";
        for (uint64_t f : first) std::cout << " " << f;
        std::cout << "\n";
    }
    return 0;
}
