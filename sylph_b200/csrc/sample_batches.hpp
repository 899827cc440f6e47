// sample_batches.hpp — how syl_query_host_samples / syl_profile_host_samples cut host-memory samples into batches that
// are staged on the device one after the other.  Host-only and free of CUDA, so that tests/cpp/sample_batches_check.cpp
// can build it with a plain C++ compiler.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

namespace syl {

// Device bytes of one batch of S samples holding `kmers` k-mers, the largest n_max, against G genomes.
//   per_kmer:   the batch's slot (hash + count, 12 B) and its share of the sort's second buffer, for both slots
//   per_sample: segment offsets, join views and row tables
//   per_hit:    the joins' per-key scratch, per k-mer of the largest sample and per sample
//   per_pair:   the joins' per-(sample, genome) scratch
//   fixed:      per batch (the sort's temporary storage)
struct BatchCost {
    uint64_t per_kmer, per_sample, per_hit, per_pair, fixed;
};

inline uint64_t batch_bytes(const BatchCost &c, uint64_t kmers, uint64_t S, uint64_t n_max, uint64_t G) {
    return c.fixed + c.per_kmer * kmers + S * (c.per_sample + c.per_hit * n_max + c.per_pair * G);
}

enum BatchPlanResult { BATCH_OK = 0, BATCH_OOM = 1, BATCH_TOO_MANY_KMERS = 2 };

// Cut samples [0, S) (sample i holds off[i + 1] - off[i] k-mers; off monotone) into contiguous batches: batch b is
// [first[b], first[b + 1]), the longest run from first[b] whose batch_bytes stays within budget / 2 (the next batch is
// staged while this one is joined, so two are live at once), whose pairs (samples x G) stay within max_pairs, whose
// k-mers stay within max_kmers and which has at most max_samples samples (0: no cap).  A sample whose pairs alone pass
// max_pairs is a batch of its own.  BATCH_OOM: sample *bad alone needs *need bytes (twice its batch_bytes) and the
// budget is smaller; BATCH_TOO_MANY_KMERS: sample *bad alone holds more than max_kmers k-mers.  S == 0 gives no batch
// (first = {0}).
inline BatchPlanResult plan_sample_batches(const uint64_t *off, uint32_t S, uint64_t G, uint64_t budget, uint64_t max_pairs,
                                           uint64_t max_kmers, uint32_t max_samples, const BatchCost &cost,
                                           std::vector<uint32_t> &first, uint32_t *bad, uint64_t *need) {
    first.assign(1, 0);
    uint32_t s0 = 0;
    uint64_t n_max = 0;
    for (uint32_t i = 0; i < S; i++) {
        const uint64_t n = off[i + 1] - off[i];
        if (n > max_kmers) { *bad = i; *need = n; return BATCH_TOO_MANY_KMERS; }
        if (2 * batch_bytes(cost, n, 1, n, G) > budget) { *bad = i; *need = 2 * batch_bytes(cost, n, 1, n, G); return BATCH_OOM; }
        const uint64_t m = std::max(n_max, n), S1 = (uint64_t)(i - s0) + 1, kmers = off[i + 1] - off[s0];
        const bool fits = 2 * batch_bytes(cost, kmers, S1, m, G) <= budget && S1 * G <= max_pairs && kmers <= max_kmers &&
                          (!max_samples || S1 <= max_samples);
        if (i > s0 && !fits) {
            first.push_back(i);
            s0 = i;
            n_max = n;
        } else {
            n_max = m;
        }
    }
    if (S) first.push_back(S);
    return BATCH_OK;
}

}  // namespace syl
