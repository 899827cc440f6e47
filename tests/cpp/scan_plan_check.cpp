// Reads commands from stdin, one per line, and prints what sylph_b200/csrc/scan_plan.hpp answers:
//   rule n_kmers n_tracked n_genomes n_samples sample_kmers one_batch pinned  -> 1 (scan) or 0 (build)
//   decide forced n_kmers n_tracked n_genomes n_samples sample_kmers one_batch pinned  -> scan_decision (forced: -1, 0, 1)
//   forced TEXT                                                         -> scan_forced("TEXT"); "-" stands for unset
//   cut G entries genomes off_0 .. off_G                                -> first genome of every chunk, then G
//   table n key_0 .. key_n-1 (sorted)                                   -> NB M dir_0 .. dir_NB fp_0 .. fp_n-1
//   const                                                               -> SCAN_MIN_ENTRIES SCAN_CHUNK
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "scan_plan.hpp"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string cmd;
        in >> cmd;
        std::ostringstream out;
        if (cmd == "rule") {
            syl::ScanShape s{};
            int one = 0, pinned = 0;
            in >> s.n_kmers >> s.n_tracked >> s.n_genomes >> s.n_samples >> s.sample_kmers >> one >> pinned;
            s.one_batch = one != 0;
            s.pinned = pinned != 0;
            out << (syl::scan_wins(s) ? 1 : 0);
        } else if (cmd == "decide") {
            syl::ScanShape s{};
            int forced = -1, one = 0, pinned = 0;
            in >> forced >> s.n_kmers >> s.n_tracked >> s.n_genomes >> s.n_samples >> s.sample_kmers >> one >> pinned;
            s.one_batch = one != 0;
            s.pinned = pinned != 0;
            out << (syl::scan_decision(s, forced) ? 1 : 0);
        } else if (cmd == "forced") {
            std::string t;
            in >> t;
            out << syl::scan_forced(t == "-" ? nullptr : t.c_str());
        } else if (cmd == "cut") {
            uint64_t G = 0, entries = 0, genomes = 0;
            in >> G >> entries >> genomes;
            std::vector<uint64_t> off(G + 1), first;
            for (uint64_t &o : off) in >> o;
            syl::cut_scan_chunks(off.data(), G, entries, genomes, first);
            for (size_t i = 0; i < first.size(); i++) out << (i ? " " : "") << first[i];
        } else if (cmd == "table") {
            uint64_t n = 0;
            in >> n;
            std::vector<uint64_t> keys(n);
            for (uint64_t &k : keys) in >> k;
            const uint64_t NB = syl::table_buckets(n), M = syl::table_mult(n ? keys[n - 1] : 0, NB);
            std::vector<uint32_t> dir(NB + 1, 0xFFFFFFFFu);
            if (!n) dir[0] = dir[1] = 0;
            for (uint64_t i = 0; i < n; i++) syl::table_dir_entries(keys.data(), n, i, M, NB, dir.data());
            out << NB << " " << M;
            for (uint32_t d : dir) out << " " << d;
            for (uint64_t k : keys) out << " " << (uint32_t)k;
        } else if (cmd == "const") {
            out << syl::SCAN_MIN_ENTRIES << " " << syl::SCAN_CHUNK;
        } else {
            continue;
        }
        std::printf("%s\n", out.str().c_str());
    }
    return 0;
}
