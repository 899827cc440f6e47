// sample_parts.hpp — how a read or pair sketch is cut into hash ranges ("parts") that each fit a device memory budget.
// Host-only and free of CUDA, so that tests/cpp/sample_parts_check.cpp can build it with a plain C++ compiler.
//
// The dedup state of a read sketch is per k-mer (src/sketch.rs:690-731; the paired rule :849-853 compares one k-mer
// within one pair), so the sketch of the hashes in [lo, hi) does not depend on any other hash.  Part p sketches the
// hashes [lo_p, hi_p) in a pass of its own over the input; the parts' sketches, in range order, concatenate into the
// one-pass sketch.  The bounds are bucket boundaries of the one-pass group map, so each part is a contiguous run of
// the post-pass groups (the first and last of them possibly holding only some of their buckets).
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

namespace syl {

constexpr uint32_t GRP_BPG = 32;   // hash buckets per read-sketch post-pass group (GroupOut in seed_kernel.cuh)
constexpr int GRP_CAP = 1024;      // most events one post-pass CTA handles in shared memory (= slot per group)
constexpr int GRP_T = 640;         // expected events per group: room in the slot for the spread of duplicate-heavy k-mers
constexpr uint32_t SAMPLE_MAX_PARTS = 64;
constexpr uint64_t SAMPLE_MAX_EVENTS = 0xFFFFFFFEull;  // a part's event array (slots + overflow list) stays below this

// Device bytes per entry of the post-pass arrays (sample.cu, SampleBuilder):
constexpr uint64_t SP_EVENT_BYTES = 32 + 4;          // begin(): EventRec + pending index, per slot and per overflow entry
// finish(): the staged (hash, count) pairs k_group_dedup writes, 8 + 4 B per slot (the exact-size result is
// SP_RESULT_BYTES).  The plan reserves twice that, as when the uniques were staged and then compacted into a second
// array: the planned part sizes, and with them the parts a budget yields, stay as they were, 12 B per slot (about 19 B
// per expected event) on the safe side.
constexpr uint64_t SP_STAGE_BYTES = 8 + 4 + 8 + 4;
constexpr uint64_t SP_GROUP_BYTES = 4 + 6 * 4 + 1;   // g_cnt; g_nuniq, g_n, uoff, fsz, foff, g_src; g_fb
// the generic path per event handed to it: the event's four words, two index and two key buffers of the radix sorts,
// the sorts' alternate buffers, uniques, run offsets and lengths, counts and the two-slot dedup set
constexpr uint64_t SP_GENERIC_BYTES = 32 + 8 + 16 + 12 + 8 + 8 + 4 + 4 + 16;
constexpr uint64_t SP_RESULT_BYTES = 8 + 4;          // the sketch: hash and count per unique k-mer
constexpr uint64_t SP_SLACK_BYTES = 16ull << 20;     // scan and sort temporaries, allocation rounding

// The one-pass group map (SampleBuilder::begin): ng groups of GRP_BPG buckets, bucket = min(mulhi(hash, Mb), nbk - 1),
// for the n_exp events expected from `bases` bases in `records` records.
struct SampleMap {
    uint64_t n_exp = 0, thr = 0, Mb = 0;
    uint32_t ng = 0, nbk = 0;
};

inline uint64_t sample_threshold(uint64_t c) { return ~0ull / c; }  // fmh_threshold (src/seeding.rs:108)

// false: 2^32 buckets or more (the map cannot be built)
inline bool sample_map(uint64_t bases, uint64_t records, int k, uint64_t c, SampleMap &m) {
    const unsigned __int128 edge = (unsigned __int128)records * (uint64_t)(k - 1);
    const uint64_t win = (unsigned __int128)bases > edge ? bases - (uint64_t)edge : 0;
    m.n_exp = win / c;
    m.thr = sample_threshold(c);
    const uint64_t g = m.n_exp / GRP_T + 1;
    if (g * GRP_BPG >= 0xFFFFFFFFull) return false;
    m.ng = (uint32_t)g;
    m.nbk = m.ng * GRP_BPG;
    const unsigned __int128 mb = ((unsigned __int128)m.nbk << 64) / ((unsigned __int128)m.thr + 1);
    m.Mb = mb > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)mb;
    return true;
}

// smallest hash of bucket b (mulhi(h, Mb) >= b), at most thr
inline uint64_t bucket_first_hash(uint32_t b, const SampleMap &m) {
    if (b == 0) return 0;
    const unsigned __int128 h = (((unsigned __int128)b << 64) + (m.Mb - 1)) / m.Mb;
    return h > (unsigned __int128)m.thr ? m.thr : (uint64_t)h;
}

// Bases that a part of hashes [lo, hi) stands for: its share of the threshold (all of them for the whole range).
inline uint64_t part_bases(uint64_t bases, uint64_t lo, uint64_t hi, uint64_t thr) {
    if (lo == 0 && hi == thr) return bases;
    return (uint64_t)((unsigned __int128)bases * (hi - lo) / thr);
}

// Overflow list of a part that stands for eb bases (SampleBuilder::begin): 1/16 of the estimate with groups, all of it
// without (SYL_SAMPLE_POSTPASS=sort).
inline uint64_t overflow_cap(uint64_t eb, uint64_t c, bool grouped) {
    uint64_t cap = eb / c + (c >> 61 ? 0 : eb / (4 * c)) + 65536;
    if (cap > eb) cap = eb + 16;
    if (grouped) cap = cap / 16 + 65536;
    return cap;
}

struct SamplePart {
    uint64_t lo = 0, hi = 0;   // hashes [lo, hi)
    uint32_t g0 = 0, ng = 0;   // groups [g0, g0 + ng) of the one-pass map (ng = 0 without groups)
    uint64_t cap = 0;          // overflow list
    uint64_t events = 0;       // slots + overflow list
    uint64_t bytes = 0;        // device bytes of the part's pass
};

inline void part_size(SamplePart &p, const SampleMap &m, uint64_t bases, uint64_t c, bool grouped) {
    const uint64_t eb = part_bases(bases, p.lo, p.hi, m.thr);
    p.cap = overflow_cap(eb, c, grouped);
    const uint64_t ng = grouped ? p.ng : 0, slots = ng * GRP_CAP, n = eb / c;
    p.events = slots + p.cap;
    // the generic path: with groups the overflow list's events are expected there, without groups (cap = every event) all
    const uint64_t generic = p.cap;
    p.bytes = p.events * SP_EVENT_BYTES + slots * SP_STAGE_BYTES + ng * SP_GROUP_BYTES + generic * SP_GENERIC_BYTES +
              (n + n / 4) * SP_RESULT_BYTES;
}

struct SamplePlan {
    SampleMap map;
    std::vector<SamplePart> parts;
    uint64_t need = 0;  // device bytes the plan needs: fixed + the largest part (or the assembled sketch)
};

enum { PLAN_OK = 0, PLAN_TOO_MANY_EVENTS = 1, PLAN_OVER_BUDGET = 2 };

// Cut [0, thr) into P parts at the bucket boundaries round(p * nbk / P).
inline void cut_parts(const SampleMap &m, uint64_t bases, uint64_t c, bool grouped, uint32_t P, SamplePlan &plan) {
    plan.parts.assign(P, SamplePart());
    for (uint32_t p = 0; p < P; p++) {
        SamplePart &s = plan.parts[p];
        const uint32_t b0 = (uint32_t)((uint64_t)m.nbk * p / P), b1 = (uint32_t)((uint64_t)m.nbk * (p + 1) / P);
        s.lo = p == 0 ? 0 : bucket_first_hash(b0, m);
        s.hi = p + 1 == P ? m.thr : bucket_first_hash(b1, m);
        s.g0 = b0 / GRP_BPG;
        s.ng = grouped ? (b1 + GRP_BPG - 1) / GRP_BPG - s.g0 : 0;
        part_size(s, m, bases, c, grouped);
    }
}

// Plan the sketch of `records` records per mate (`mates` of them per record) holding `bases` bases in all, within
// `budget` device bytes of which `fixed` are taken already (staging rings, staged 2-bit input).  forced > 0: exactly
// that many parts (at most one per bucket), whatever the budget.  Otherwise the fewest parts, at most
// SAMPLE_MAX_PARTS, whose largest pass fits.  With more than one part the parts' sketches wait in host memory and the
// device ends up holding the assembled sketch.
inline int plan_sample_parts(uint64_t bases, uint64_t records, int mates, int k, uint64_t c, bool grouped,
                             uint64_t budget, uint64_t fixed, uint32_t forced, SamplePlan &plan) {
    plan = SamplePlan();
    if (!sample_map(bases, records * (uint64_t)mates, k, c, plan.map)) return PLAN_TOO_MANY_EVENTS;
    const SampleMap &m = plan.map;
    const uint64_t assembled = (m.n_exp + m.n_exp / 4) * SP_RESULT_BYTES;
    auto need = [&]() {
        uint64_t big = 0;
        bool fits = true;
        for (const SamplePart &s : plan.parts) {
            big = std::max(big, s.bytes);
            fits = fits && s.events < SAMPLE_MAX_EVENTS;
        }
        if (plan.parts.size() > 1) big = std::max(big, assembled);
        plan.need = fixed + SP_SLACK_BYTES + big;
        return fits;
    };
    if (forced) {
        cut_parts(m, bases, c, grouped, std::min<uint32_t>(forced, m.nbk), plan);
        return need() ? PLAN_OK : PLAN_TOO_MANY_EVENTS;
    }
    bool any_fits = false;
    for (uint32_t P = 1; P <= std::min<uint32_t>(SAMPLE_MAX_PARTS, m.nbk); P++) {
        cut_parts(m, bases, c, grouped, P, plan);
        const bool fits = need();
        any_fits = any_fits || fits;
        if (fits && plan.need <= budget) return PLAN_OK;
    }
    return any_fits ? PLAN_OVER_BUDGET : PLAN_TOO_MANY_EVENTS;
}

}  // namespace syl
