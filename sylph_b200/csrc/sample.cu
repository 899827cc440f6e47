// sample.cu — sample (read) sketch: seeding survivors -> FxHashMap<Kmer,u32> equivalent.
//
// Replaces the per-record loop of sketch_sequences_needle (src/sketch.rs:917-947):
//   pair_kmer_single (:624-656), extract_markers (:928), and for every survivor
//   dup_removal_lsh_full_exact(.., Some(MAX_DEDUP_COUNT)) (:690-731).
//
// The reference walks reads in file order and keeps ONE global exact set S of (kmer, pair-key)
// plus the count map.  S is keyed by the k-mer, so the state of different k-mers never
// interacts; only the order of the events OF ONE k-mer matters, and that order is read order.
// Device formulation: every survivor is an event (hash, read index, p0, p1), written by the
// seeding kernel itself; the events are partitioned by hash bucket, a CTA groups the events of
// ~25 consecutive buckets by k-mer in shared memory and one thread replays the state machine
// of one k-mer over its first events in read order (after four counted events every further
// event counts).  Groups that do not fit take the generic path: two stable LSD radix sorts by
// (hash, read index) and one thread per (contiguous) k-mer segment.  Within one read the order
// of repeated k-mers is irrelevant (identical events; the second is a duplicate either way).
// Read pairs (sketch_pair_sequences with --fpr 0, src/sketch.rs:771-895) take the same groups with their own
// per-k-mer rule (k_group_dedup<true>), and the same generic path with k_dedup_paired.
#include <cub/cub.cuh>

#include <chrono>
#include <cstdlib>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "common.cuh"
#include "host_pack.hpp"
#include "ingest.hpp"
#include "scan.cuh"

namespace syl {

// pair_kmer_single (src/sketch.rs:624-656): four 16-base keys sampled at even/odd offsets from
// the read start and from the middle.  len > 400 (src/sketch.rs:923) or len < 66 (:627) => None.
// The seeding kernel computes the keys itself from its packed tile whenever the read's first 32 bases
// and the 32 bases from its middle are inside the tile; k_events_fix below handles the reads cut by a
// tile edge.  One thread per such event.  ASCII input: the 32 bytes a key pair is drawn from are
// fetched as nine aligned 32-bit words and realigned with funnel shifts; even / odd bytes are
// separated with PRMT and mapped through four pre-shifted copies of the exact BYTE_TO_SEQ table in
// shared memory.  2-bit input: three words, one funnel extract, even / odd fields compressed.
constexpr int EV_THREADS = 128;

__device__ __forceinline__ void load32_unaligned(const uint8_t *p, uint32_t x[8]) {
    const uintptr_t ad = reinterpret_cast<uintptr_t>(p);
    const uint32_t *w = reinterpret_cast<const uint32_t *>(ad & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(ad & 3u) * 8u;
    uint32_t v[9];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = __ldg(w + i);
    v[8] = sh ? __ldg(w + 8) : 0u;  // an aligned word holding a valid byte never leaves the buffer's last word
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = __funnelshift_r(v[i], v[i + 1], sh);
}

// 16 bytes picked by `sel` (0x6420 = even, 0x7531 = odd) out of 32 -> 16 two-bit codes, MSB-first
__device__ __forceinline__ uint32_t pack16(const uint32_t x[8], uint32_t sel, const uint8_t (*lut)[256]) {
    uint32_t out = 0;
#pragma unroll
    for (int m = 0; m < 4; m++) {
        const uint32_t e = __byte_perm(x[2 * m], x[2 * m + 1], sel);
        const uint32_t g = ((uint32_t)lut[0][e & 0xFFu] | (uint32_t)lut[1][(e >> 8) & 0xFFu] |
                            (uint32_t)lut[2][(e >> 16) & 0xFFu]) | (uint32_t)lut[3][e >> 24];
        out = (out << 8) | g;
    }
    return out;
}

// 32 bases starting at base `a` of a 2-bit packed buffer of n_words words -> 64 bits, MSB-first
__device__ __forceinline__ uint64_t packed64(const uint32_t *__restrict__ packed, uint64_t n_words, uint64_t a) {
    const uint64_t w = a >> 4;
    const uint32_t sh = (uint32_t)(a & 15u) * 2u;
    const uint32_t v0 = __ldg(packed + w), v1 = w + 1 < n_words ? __ldg(packed + w + 1) : 0u,
                   v2 = w + 2 < n_words ? __ldg(packed + w + 2) : 0u;
    return ((uint64_t)__funnelshift_l(v1, v0, sh) << 32) | __funnelshift_l(v2, v1, sh);
}

// Events pend[*p_begin .. *p_end) (indices into ev) are the pending events of one batch of records [rec_base, ..), and
// arrive with recflag = record << 1 | EV_PENDING.  The keys are built from 32 bases at the record's start and 32 more:
//   single-end: from the middle of the read (pair_kmer_single); recflag = read << 1 | NO_PAIR as the seeding kernel set it.
//   read pairs (src/sketch.rs:658-688 pair_kmer): from the start of mate 2, so every event of the pair carries the same
//       keys; recflag = pair << 2 | mate << 1 | NO_PAIR (a mate shorter than 33 bp, or --no-dedup).  The batch's mate-2
//       events start at pend[*p_mate2].
template <bool PACKED, bool PAIRED>
__global__ void __launch_bounds__(EV_THREADS)
k_events_fix(EventRec *__restrict__ ev, const uint32_t *__restrict__ pend, const unsigned long long *__restrict__ p_begin,
             const unsigned long long *__restrict__ p_mate2, const unsigned long long *__restrict__ p_end, uint64_t ev_cap,
             const Mate m1, const Mate m2, uint64_t rec_base, int no_dedup) {
    __shared__ uint8_t lut[4][256];
    if (!PACKED) {
        for (int i = threadIdx.x; i < 256; i += EV_THREADS) {
            const uint32_t code = byte_to_seq((uint32_t)i);
            lut[0][i] = (uint8_t)(code << 6);
            lut[1][i] = (uint8_t)(code << 4);
            lut[2][i] = (uint8_t)(code << 2);
            lut[3][i] = (uint8_t)code;
        }
        __syncthreads();
    }
    const Mate &ms = PAIRED ? m2 : m1;  // where the second 32 bases come from
    const uint64_t i0 = *p_begin, i1 = *p_end, i2 = PAIRED ? *p_mate2 : i1;
    for (uint64_t i = i0 + (uint64_t)blockIdx.x * EV_THREADS + threadIdx.x; i < i1; i += (uint64_t)gridDim.x * EV_THREADS) {
        const uint32_t ei = pend[i];
        if (ei >= ev_cap) continue;
        EventRec *e = ev + ei;
        const uint64_t rf = e->recflag & ~EV_PENDING, rec = (rf >> 1) - rec_base;
        // __ldg: Mate's pointers are not __restrict__, and the plain loads made the pair kernel 2.5 % slower (H100, 700 W)
        auto start = [rec](const Mate &m, uint64_t r) { return __ldg(m.off + rec + r) - m.off_bias; };
        const uint64_t a = start(m1, 0), L = start(m1, 1) - a;
        uint64_t b = a + L / 2;
        bool has = true;
        if (PAIRED) {
            b = start(ms, 0);
            const uint64_t L2 = start(ms, 1) - b;
            has = !no_dedup && L >= 33 && L2 >= 33;  // 2 * 16 + 1 (:660)
        }
        uint64_t p0 = 0, p1 = 0;
        if (has) {
            uint32_t f, g, r, t;
            if (!PACKED) {
                uint32_t x[8];
                load32_unaligned(m1.bases + a, x);
                f = pack16(x, 0x6420, lut); g = pack16(x, 0x7531, lut);
                load32_unaligned(ms.bases + b, x);
                r = pack16(x, 0x6420, lut); t = pack16(x, 0x7531, lut);
            } else {
                const uint64_t x = packed64(m1.packed, (m1.nb + 15) / 16, a), y = packed64(ms.packed, (ms.nb + 15) / 16, b);
                f = even_fields(x); g = even_fields(x << 2);
                r = even_fields(y); t = even_fields(y << 2);
            }
            p0 = ((uint64_t)f << 32) | r;  // doublepairs.0 = [kmer_f, kmer_r]
            p1 = ((uint64_t)g << 32) | t;  // doublepairs.1 = [kmer_g, kmer_t]
        }
        e->recflag = PAIRED ? ((rf >> 1) << 2) | ((uint64_t)(i >= i2) << 1) | (has ? 0ull : NO_PAIR) : rf;
        e->p0 = p0;
        e->p1 = p1;
    }
}

// One WARP replays dup_removal_lsh_full_exact(.., threshold None) (src/sketch.rs:690-731, call :829-865) for one
// k-mer of a paired sample: events sorted by (pair, mate); a mate-2 event whose k-mer also occurs in mate 1 of the
// same pair is skipped (:849-853); the dedup set never stops growing (no MAX_DEDUP_COUNT), membership is tested by
// the 32 lanes in parallel.  set[] is this segment's private slice of a global scratch array (2 slots per event).
__global__ void k_dedup_paired(const uint64_t *__restrict__ seg_off, const uint32_t *__restrict__ seg_len, uint64_t n_seg,
                               const uint32_t *__restrict__ order, const uint64_t *__restrict__ recflag,
                               const uint64_t *__restrict__ p0, const uint64_t *__restrict__ p1, int no_dedup,
                               uint64_t *__restrict__ set, uint32_t *__restrict__ count, unsigned long long *__restrict__ n_dup) {
    const uint64_t s = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (s >= n_seg) return;
    const uint64_t start = seg_off[s];
    const uint32_t len = seg_len[s];
    uint64_t *S = set + 2 * start;
    uint32_t nset = 0, c = 0, dups = 0;
    uint64_t last_m1_pair = 0xFFFFFFFFFFFFFFFFull;
    for (uint32_t e = 0; e < len; e++) {
        const uint32_t evi = order[start + e];
        const uint64_t rf = recflag[evi];
        const uint64_t pair = rf >> 2;
        if (((rf >> 1) & 1ull) == 0) last_m1_pair = pair;
        else if (pair == last_m1_pair) continue;  // temp_vec1.contains(km)
        if (no_dedup || (rf & NO_PAIR)) { c++; continue; }
        const uint64_t a = p0[evi], b = p1[evi];
        bool fa = false, fb = false;
        for (uint32_t q = lane; q < nset; q += 32) { const uint64_t v = S[q]; fa |= v == a; fb |= v == b; }
        fa = __any_sync(0xffffffffu, fa);
        fb = __any_sync(0xffffffffu, fb) || (!fa && a == b);  // the second look-up sees the first key's insertion
        if (lane == 0) {
            if (!fa) S[nset] = a;
            if (!fb) S[nset + (fa ? 0 : 1)] = b;
        }
        nset += (fa ? 0u : 1u) + (fb ? 0u : 1u);
        __syncwarp();
        if ((fa || fb) && c > 0) dups++; else c++;
    }
    if (lane == 0) {
        count[s] = c;
        if (dups) atomicAdd(n_dup, (unsigned long long)dups);
    }
}

__global__ void k_unpack_events(const EventRec *__restrict__ ev, uint64_t n, uint64_t *__restrict__ hash,
                                uint64_t *__restrict__ recflag, uint64_t *__restrict__ p0, uint64_t *__restrict__ p1) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const EventRec r = ev[i];
    hash[i] = r.hash; recflag[i] = r.recflag; p0[i] = r.p0; p1[i] = r.p1;
}

__global__ void k_iota(uint32_t *idx, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (uint32_t)i;
}

template <typename T>
__global__ void k_gather(const T *__restrict__ src, const uint32_t *__restrict__ idx, T *__restrict__ dst, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[idx[i]];
}

// One thread replays dup_removal_lsh_full_exact (src/sketch.rs:690-731) for one k-mer.
// set[] is this segment's private slice of a global scratch array (2 slots per event).
__global__ void k_dedup(const uint64_t *__restrict__ seg_off, const uint32_t *__restrict__ seg_len, uint64_t n_seg,
                        const uint32_t *__restrict__ order, const uint64_t *__restrict__ recflag,
                        const uint64_t *__restrict__ p0, const uint64_t *__restrict__ p1,
                        uint64_t *__restrict__ set, uint32_t *__restrict__ count,
                        unsigned long long *__restrict__ n_dup) {
    uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const uint64_t start = seg_off[s];
    const uint32_t len = seg_len[s];
    if (len == 1) {  // first occurrence is never a duplicate (c == 0)
        count[s] = 1;
        return;
    }
    uint64_t *S = set + 2 * start;
    uint32_t nset = 0, c = 0, dups = 0;
    for (uint32_t e = 0; e < len; e++) {
        if (c >= 4u) {  // MAX_DEDUP_COUNT (src/constants.rs:14): dedup is off from here on
            c += len - e;
            break;
        }
        const uint32_t ev = order[start + e];
        if (recflag[ev] & NO_PAIR) {
            c++;
            continue;
        }
        const uint64_t a = p0[ev], b = p1[ev];
        bool ret = false, found = false;
        for (uint32_t q = 0; q < nset; q++) found |= (S[q] == a);
        if (found) ret = c > 0; else S[nset++] = a;
        found = false;
        for (uint32_t q = 0; q < nset; q++) found |= (S[q] == b);
        if (found) ret = ret || c > 0; else S[nset++] = b;
        if (ret) dups++; else c++;
    }
    count[s] = c;
    if (dups) atomicAdd(n_dup, (unsigned long long)dups);
}


// ------------------------------------------------------------------------------------------------
// Post-pass, primary path: MSD bucket partition + CTA-local grouping + fused run-length / dedup.
//   the seeding kernel's flush (GroupOut, seed_kernel.cuh) : writes every event into the slot of its
//       group g = bucket / GRP_BPG, bucket = min(mulhi(hash, Mb), nbk - 1) (monotone in the hash, uniform
//       because hashes are uniform below thr); the groups are fixed in begin() at ~GRP_T expected events
//   k_group_dedup : one CTA per group (<= slot events) groups the events by k-mer in shared memory,
//       replays dup_removal_lsh_full_exact per k-mer and writes the group's sorted (hash, count) pairs into
//       its slot of the staging arrays
//   k_compact_uniq : staged pairs -> the exact-size result; buckets are monotone in the hash and every
//       group is sorted, so the result is globally sorted without a merge.
// Groups that do not fit (heavy-hitter k-mers: more events than the slot, the rest in the overflow list)
// or whose dedup set outgrows the per-thread buffer are handed to the generic radix-sort path below, and
// k_compact_uniq takes their uniques from there.
constexpr int GRP_THREADS = 256;
// GRP_CAP (slot per group) and GRP_T (expected events per group): sample_parts.hpp

__device__ __forceinline__ uint32_t bucket_of(uint64_t h, uint64_t Mb, uint32_t nbk) {
    const uint32_t b = (uint32_t)__umul64hi(h, Mb);
    return b < nbk ? b : nbk - 1;
}

// One CTA per group (<= slot events, GRP_BPG consecutive buckets). Shared-memory traffic is what
// bounds this kernel, so instead of sorting all events (a 128-bit-key bitonic sort was 4x slower)
// it (1) groups equal hashes with an open-addressing table, (2) replays
// dup_removal_lsh_full_exact on each k-mer's first events in read order, (3) orders the resulting
// unique (hash, count) pairs: the group's buckets are already monotone in the hash, so a pair's
// position is its bucket's offset plus its rank among the ~10 pairs of the same bucket.
// Table slots: a group holds at most GRP_CAP events and usually far fewer distinct k-mers (≈220 of ≈640 events on
// bench.py's sample, ≈640 on reads without repeats), so 1024 slots keep the probes short while the smaller table
// lets more CTAs share an SM; with at most GRP_CAP distinct hashes a free or equal slot always exists.
constexpr int GRP_SLOTS = 1024;
constexpr int GRP_SELECT_STEPS = 64;  // selection steps before a duplicate-heavy k-mer goes to the generic path

// Single-end groups keep the pair keys in global memory: only the k-mers with two or more events read them (the
// sectors are still in L2), and the 16 KB less (28 KB in all) lets 7 CTAs share an SM.  Read pairs compare every key
// of a k-mer with every other one, so their groups stage the keys.
template <bool PAIRED>
struct GroupSmem {
    unsigned long long ht[GRP_SLOTS];  //  8 KB  hash per slot
    uint64_t rf[GRP_CAP];              //  8 KB  recflag per event
    uint64_t p0[PAIRED ? GRP_CAP : 1]; //  8 KB  first pair key per event (PAIRED)
    uint64_t p1[PAIRED ? GRP_CAP : 1]; //  8 KB  second pair key per event (PAIRED)
    uint16_t scnt[GRP_SLOTS];          //  2 KB  events per slot, then fill cursor, then the k-mer's count
    uint16_t soff[GRP_SLOTS + 2];      //  2 KB  exclusive scan of scnt
    uint16_t ev_slot[GRP_CAP];         //  2 KB  slot per event | after the member fill: 2 x GRP_BPG bucket counters / offsets
    uint16_t member[GRP_CAP];          //  2 KB  event indices grouped by slot
    uint16_t occ[GRP_CAP];             //  2 KB  occupied slots, compacted
    uint32_t wtot[GRP_THREADS / 32], wocc[GRP_THREADS / 32];
    uint32_t overflow, dups, nlong;
    uint16_t longs[GRP_CAP / 2];      //  1 KB  slots of k-mers that need the warp-cooperative replay
};

// Read pairs: dup_removal_lsh_full_exact with threshold None (src/sketch.rs:829-865) for one k-mer whose len events
// are S.member[a0 ..), recflag = pair << 2 | mate << 1 | NO_PAIR.  There is no MAX_DEDUP_COUNT, so every event is
// tested, but nothing has to be replayed in order: the dedup set an event sees is the keys of the earlier paired
// events that were not skipped, "earlier" is a compare of (recflag, event index), and c > 0 means that any event
// that was not skipped comes earlier.  Two passes over the k-mer's events, each event against all others; the
// caller's threads take events first, first + step, .. (one thread: 0, 1; a warp: lane, 32).
constexpr uint64_t EV_SKIP = 1ull << 63;   // mate-2 event whose k-mer mate 1 of the same pair holds too (:849-853)
constexpr uint32_t GRP_PAIR_THREAD = 8;    // events up to which one thread does the k-mer's len^2 compares; a warp beyond

__device__ __forceinline__ void pair_mark_skipped(GroupSmem<true> &S, uint32_t a0, uint32_t len, uint32_t first, uint32_t step) {
    for (uint32_t e = first; e < len; e += step) {
        const uint32_t m = S.member[a0 + e];
        const uint64_t rf = S.rf[m];
        if (!(rf & 2ull)) continue;
        bool in_mate1 = false;
        for (uint32_t q = 0; q < len; q++) in_mate1 |= S.rf[S.member[a0 + q]] == (rf ^ 2ull);  // NO_PAIR is the pair's
        if (in_mate1) S.rf[m] = rf | EV_SKIP;
    }
}

__device__ __forceinline__ void pair_count(const GroupSmem<true> &S, uint32_t a0, uint32_t len, uint32_t first, uint32_t step,
                                           uint32_t &c, uint32_t &dups) {
    for (uint32_t e = first; e < len; e += step) {
        const uint32_t m = S.member[a0 + e];
        const uint64_t rf = S.rf[m];
        if (rf & EV_SKIP) continue;
        if (rf & NO_PAIR) { c++; continue; }  // a mate under 33 bp, or --no-dedup
        const uint64_t ka = S.p0[m], kb = S.p1[m];
        bool earlier = false, hit = false;
        for (uint32_t q = 0; q < len; q++) {
            const uint32_t mq = S.member[a0 + q];
            const uint64_t rq = S.rf[mq];
            if ((rq & EV_SKIP) || !(rq < rf || (rq == rf && mq < m))) continue;
            earlier = true;
            if (rq & NO_PAIR) continue;
            const uint64_t qa = S.p0[mq], qb = S.p1[mq];
            hit |= ka == qa || ka == qb || kb == qa || kb == qb;
        }
        // the second look-up sees the first key's insertion: ka == kb is a hit, a duplicate once c > 0 (:704-722)
        if (hit || (ka == kb && earlier)) dups++; else c++;
    }
}

// Single-end: 28 KB of shared memory and at most 32 registers, so 7 CTAs share an SM; pairs: 44 KB and 48, 5 CTAs.
template <bool PAIRED>
__global__ void __launch_bounds__(GRP_THREADS, PAIRED ? 5 : 7)
k_group_dedup(const EventRec *__restrict__ ev, const uint32_t *__restrict__ g_cnt, uint32_t slot, uint64_t Mb, uint32_t nbk,
              uint32_t g0, int no_dedup, uint64_t *__restrict__ st_hash, uint32_t *__restrict__ st_cnt,
              uint32_t *__restrict__ g_nuniq, uint32_t *__restrict__ g_n,
              uint8_t *__restrict__ g_fallback, unsigned long long *__restrict__ counters) {
    extern __shared__ __align__(16) uint8_t grp_smem_raw[];
    GroupSmem<PAIRED> &S = *reinterpret_cast<GroupSmem<PAIRED> *>(grp_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t g = blockIdx.x;
    if (tid == 0) {
        S.overflow = 0;
        S.dups = 0;
        S.nlong = 0;
    }
    const uint32_t e0 = g * slot, bf = (g0 + g) * GRP_BPG;  // g0: first group of the sample's part (sample_parts.hpp)
    const uint32_t n_all = g_cnt[g], n = min(n_all, slot);  // events past the slot are in the overflow list
    // pair keys of event m of the group (single-end: from global memory, last use)
    auto keys = [&](uint32_t m, uint64_t &ka, uint64_t &kb) {
        if constexpr (PAIRED) { ka = S.p0[m]; kb = S.p1[m]; return; }
        const uint4 k = __ldcs(reinterpret_cast<const uint4 *>(ev + e0 + m) + 1);
        ka = ((uint64_t)k.y << 32) | k.x;
        kb = ((uint64_t)k.w << 32) | k.z;
    };
    // a group that falls back hands its slotted events to the generic path; their number is summed for the host
    auto leave = [&](bool fallback) {
        g_nuniq[g] = 0;
        g_fallback[g] = fallback;
        if (fallback) atomicAdd(counters + CNT_FALLBACK_TOTAL, (unsigned long long)n);
    };
    if (tid == 0) g_n[g] = n;
    if (n == 0 || n_all > slot) { if (tid == 0) leave(n != 0); return; }
    // (1) stage the events, group equal hashes: slot per event, events per slot.  Every load of the thread's events is
    //     in flight before the table is cleared, so the CTA waits for memory once, not once per event.
    constexpr int EPT = GRP_CAP / GRP_THREADS;  // events per thread (n <= slot <= GRP_CAP)
    static_assert(GRP_CAP % GRP_THREADS == 0, "whole events per thread");
    uint4 ea[EPT], eb[PAIRED ? EPT : 1];
#pragma unroll
    for (int j = 0; j < EPT; j++) {
        const uint32_t i = tid + j * GRP_THREADS;
        if (i < n) {
            const uint4 *src = reinterpret_cast<const uint4 *>(ev + e0 + i);
            if constexpr (PAIRED) {
                ea[j] = __ldcs(src);  // read once
                eb[j] = __ldcs(src + 1);
            } else {
                ea[j] = __ldg(src);  // the keys of the same sector may be read in (2)
            }
        }
    }
    for (int i = tid; i < GRP_SLOTS; i += GRP_THREADS) { S.ht[i] = 0xFFFFFFFFFFFFFFFFull; S.scnt[i] = 0; }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < EPT; j++) {
        const uint32_t i = tid + j * GRP_THREADS;
        if (i >= n) break;
        const uint4 a = ea[j];
        const unsigned long long h = ((unsigned long long)a.y << 32) | a.x;
        S.rf[i] = ((uint64_t)a.w << 32) | a.z;
        if constexpr (PAIRED) {
            const uint4 b = eb[j];
            S.p0[i] = ((uint64_t)b.y << 32) | b.x;
            S.p1[i] = ((uint64_t)b.w << 32) | b.z;
        }
        uint32_t sl = (uint32_t)(h ^ (h >> 23)) & (GRP_SLOTS - 1);
        for (;;) {
            const unsigned long long prev = atomicCAS(&S.ht[sl], 0xFFFFFFFFFFFFFFFFull, h);
            if (prev == 0xFFFFFFFFFFFFFFFFull || prev == h) break;
            sl = (sl + 1) & (GRP_SLOTS - 1);
        }
        S.ev_slot[i] = (uint16_t)sl;
        atomicAdd(reinterpret_cast<unsigned int *>(S.scnt) + (sl >> 1), (sl & 1) ? 0x10000u : 1u);  // u16 counters, n <= 1024
    }
    __syncthreads();
    // exclusive scans over the slots: events per slot -> soff, occupied slots -> occ[]
    uint32_t nu;
    {
        constexpr int PER = GRP_SLOTS / GRP_THREADS;
        uint32_t loc[PER], tot = 0, oc = 0;
#pragma unroll
        for (int e = 0; e < PER; e++) { loc[e] = S.scnt[tid * PER + e]; tot += loc[e]; oc += loc[e] ? 1u : 0u; }
        uint32_t inc = tot, oinc = oc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, inc, d), u = __shfl_up_sync(0xffffffffu, oinc, d);
            if (lane >= d) { inc += t; oinc += u; }
        }
        if (lane == 31) { S.wtot[wid] = inc; S.wocc[wid] = oinc; }
        __syncthreads();
        uint32_t base = inc - tot, obase = oinc - oc, ototal = 0;
#pragma unroll
        for (int w = 0; w < GRP_THREADS / 32; w++) { if (w < wid) { base += S.wtot[w]; obase += S.wocc[w]; } ototal += S.wocc[w]; }
        nu = ototal;
#pragma unroll
        for (int e = 0; e < PER; e++) {
            S.soff[tid * PER + e] = (uint16_t)base;
            base += loc[e];
            if (loc[e]) S.occ[obase++] = (uint16_t)(tid * PER + e);
        }
        if (tid == GRP_THREADS - 1) S.soff[GRP_SLOTS] = (uint16_t)base;
        __syncthreads();
#pragma unroll
        for (int e = 0; e < PER; e++) S.scnt[tid * PER + e] = 0;  // reused as fill cursors
        __syncthreads();
    }
    for (uint32_t i = tid; i < n; i += GRP_THREADS) {
        const uint32_t sl = S.ev_slot[i];
        const unsigned int old = atomicAdd(reinterpret_cast<unsigned int *>(S.scnt) + (sl >> 1), (sl & 1) ? 0x10000u : 1u);
        const uint32_t k = (sl & 1) ? (old >> 16) : (old & 0xFFFFu);
        S.member[S.soff[sl] + k] = (uint16_t)i;
    }
    __syncthreads();
    // (2) replay dup_removal_lsh_full_exact (src/sketch.rs:690-731) per k-mer; the count lands in scnt.
    //     One thread per k-mer, registers only: a single pass over the k-mer's events keeps the four
    //     smallest (read index, event) keys; those four are replayed in order.  The dedup set at any
    //     point is simply "every pair key of the earlier paired events", so membership is a compare
    //     against the earlier events' keys and nothing has to be inserted.  Four counted events reach
    //     MAX_DEDUP_COUNT (src/constants.rs:14), after which every event counts.  Only a k-mer that
    //     has more than four events AND a duplicate among the first four needs more; it is queued
    //     for the warp-cooperative path below.
    //     The thread also counts its k-mer into its bucket (local index) for the output ordering.
    //     PAIRED: pair_mark_skipped / pair_count instead, by this thread up to GRP_PAIR_THREAD events, by a warp
    //     beyond; a group of pairs leaves the kernel only when it is past its slot.
    uint16_t *lb_cnt = S.ev_slot, *lb_off = S.ev_slot + GRP_BPG;  // ev_slot is dead: 2 x GRP_BPG u16
    if (tid < (int)GRP_BPG) lb_cnt[tid] = 0;
    __syncthreads();
    uint32_t my_dups = 0;
    for (uint32_t u = tid; u < nu; u += GRP_THREADS) {
        const uint32_t sl = S.occ[u];
        const uint32_t a0 = S.soff[sl], len = S.soff[sl + 1] - a0;
        {
            const uint32_t lb = bucket_of(S.ht[sl], Mb, nbk) - bf;
            atomicAdd(reinterpret_cast<unsigned int *>(lb_cnt) + (lb >> 1), (lb & 1) ? 0x10000u : 1u);
        }
        uint32_t c = 0;
        if constexpr (PAIRED) {
            if (len > GRP_PAIR_THREAD) { S.longs[atomicAdd(&S.nlong, 1u)] = (uint16_t)sl; continue; }
            if (len == 1) c = 1;
            else { pair_mark_skipped(S, a0, len, 0, 1); pair_count(S, a0, len, 0, 1, c, my_dups); }
        } else if (no_dedup || len == 1) {
            c = len;  // a first occurrence is never a duplicate (c == 0)
        } else {
            constexpr uint64_t INF = 0xFFFFFFFFFFFFFFFFull;
            uint64_t k0 = INF, k1 = INF, k2 = INF, k3 = INF;  // (recflag << 10 | event) ascending
            for (uint32_t e = 0; e < len; e++) {
                const uint32_t m = S.member[a0 + e];
                uint64_t key = (S.rf[m] << 10) | m;
                if (key < k3) {
                    k3 = key;
                    if (k3 < k2) { const uint64_t t = k2; k2 = k3; k3 = t; }
                    if (k2 < k1) { const uint64_t t = k1; k1 = k2; k2 = t; }
                    if (k1 < k0) { const uint64_t t = k0; k0 = k1; k1 = t; }
                }
            }
            const uint64_t ks[4] = {k0, k1, k2, k3};
            uint64_t A[4], B[4];
            bool paired[4];
            uint32_t dups = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                paired[j] = false;
                A[j] = B[j] = 0;
                if (ks[j] == INF) continue;  // len < 4
                const uint32_t m = (uint32_t)ks[j] & 1023u;
                if ((ks[j] >> 10) & NO_PAIR) { c++; continue; }
                uint64_t ka, kb;
                keys(m, ka, kb);
                bool found = (kb == ka);
#pragma unroll
                for (int i = 0; i < j; i++)
                    found |= paired[i] && (ka == A[i] || ka == B[i] || kb == A[i] || kb == B[i]);
                paired[j] = true; A[j] = ka; B[j] = kb;
                // found on the SECOND key only because it equals the first does not make a duplicate
                // of an earlier read, but sketch.rs:704-722 still returns true when cur > 0
                if (found && c > 0) dups++; else c++;
            }
            if (len > 4u) {
                if (c >= 4u) c += len - 4u;
                else {  // a duplicate among the first four: replay the whole k-mer cooperatively
                    const uint32_t li = atomicAdd(&S.nlong, 1u);
                    S.longs[li] = (uint16_t)sl;
                    continue;
                }
            }
            my_dups += dups;
        }
        S.scnt[sl] = (uint16_t)c;  // c <= len <= GRP_CAP
    }
    __syncthreads();
    for (uint32_t li = wid; li < S.nlong; li += GRP_THREADS / 32) {
        const uint32_t sl = S.longs[li];
        const uint32_t a0 = S.soff[sl], len = S.soff[sl + 1] - a0;
        if constexpr (PAIRED) {
            uint32_t c = 0, dups = 0;
            pair_mark_skipped(S, a0, len, lane, 32);
            __syncwarp();
            pair_count(S, a0, len, lane, 32, c, dups);
            c = __reduce_add_sync(0xffffffffu, c);
            dups = __reduce_add_sync(0xffffffffu, dups);
            if (lane == 0) { S.scnt[sl] = (uint16_t)c; my_dups += dups; }
            continue;
        }
        uint32_t c = 0, done = 0, nset = 0;
        uint64_t last_key = 0, dset = 0;  // lane q keeps dedup-set entry q in `dset` (32 entries, then the group falls back)
        uint32_t last_m = 0;
        bool first = true;
        while (done < len) {
            if (c >= 4u) { c += len - done; break; }  // MAX_DEDUP_COUNT
            if (done >= (uint32_t)GRP_SELECT_STEPS) { if (lane == 0) S.overflow = 1; break; }  // duplicate-heavy
            // next event after (last_key, last_m) in (read index, event index) order
            uint64_t best = 0xFFFFFFFFFFFFFFFFull;
            uint32_t bm = 0xFFFFFFFFu;
            for (uint32_t e = lane; e < len; e += 32) {
                const uint32_t m = S.member[a0 + e];
                const uint64_t key = S.rf[m];
                const bool after = first || key > last_key || (key == last_key && m > last_m);
                if (after && (key < best || (key == best && m < bm))) { best = key; bm = m; }
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) {
                const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, d);
                const uint32_t om = __shfl_xor_sync(0xffffffffu, bm, d);
                if (ok < best || (ok == best && om < bm)) { best = ok; bm = om; }
            }
            first = false; last_key = best; last_m = bm; done++;
            if (best & NO_PAIR) { c++; continue; }
            uint64_t ka, kb;
            keys(bm, ka, kb);
            const bool in_a = __any_sync(0xffffffffu, lane < (int)nset && dset == ka);
            bool ret = in_a && c > 0;
            if (!in_a) { if (lane == (int)nset) dset = ka; nset++; }
            const bool in_b = __any_sync(0xffffffffu, lane < (int)nset && lane < 32 && dset == kb);
            if (in_b) ret = ret || c > 0;
            else { if (lane == (int)nset) dset = kb; nset++; }
            if (nset > 32u) { if (lane == 0) S.overflow = 1; break; }
            if (ret) { if (lane == 0) my_dups++; } else c++;
        }
        if (lane == 0) S.scnt[sl] = (uint16_t)c;
    }
    if (my_dups) atomicAdd(&S.dups, my_dups);
    __syncthreads();
    if (S.overflow) { if (tid == 0) leave(true); return; }
    // (3) output order: lb_cnt holds the k-mers per bucket (counted in (2)); the group's sorted uniques go to its slot.
    {
        uint16_t *list = S.member;  // event grouping is dead: k-mer slots ordered by bucket
        static_assert(GRP_BPG == 32, "one lane per bucket");
        if (wid == 0) {  // exclusive scan of lb_cnt -> lb_off, counters reset as cursors
            const uint32_t v = lb_cnt[lane];
            uint32_t inc = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t; }
            lb_off[lane] = (uint16_t)(inc - v);
            lb_cnt[lane] = 0;
        }
        __syncthreads();
        for (uint32_t u = tid; u < nu; u += GRP_THREADS) {
            const uint32_t sl = S.occ[u];
            const uint32_t lb = bucket_of(S.ht[sl], Mb, nbk) - bf;
            const unsigned int old = atomicAdd(reinterpret_cast<unsigned int *>(lb_cnt) + (lb >> 1), (lb & 1) ? 0x10000u : 1u);
            list[lb_off[lb] + ((lb & 1) ? (old >> 16) : (old & 0xFFFFu))] = (uint16_t)sl;
        }
        __syncthreads();
        for (uint32_t u = tid; u < nu; u += GRP_THREADS) {
            const uint32_t sl = S.occ[u];
            const unsigned long long h = S.ht[sl];
            const uint32_t lb = bucket_of(h, Mb, nbk) - bf;
            const uint32_t q0 = lb_off[lb], q1 = q0 + ((lb & 1) ? (reinterpret_cast<unsigned int *>(lb_cnt)[lb >> 1] >> 16)
                                                                : (reinterpret_cast<unsigned int *>(lb_cnt)[lb >> 1] & 0xFFFFu));
            uint32_t r = 0;
            for (uint32_t q = q0; q < q1; q++) r += (S.ht[list[q]] < h) ? 1u : 0u;
            st_hash[e0 + q0 + r] = h;
            st_cnt[e0 + q0 + r] = S.scnt[sl];
        }
    }
    if (tid == 0) {
        g_nuniq[g] = nu;
        g_fallback[g] = 0;
        atomicAdd(counters + CNT_UNIQ_TOTAL, (unsigned long long)nu);
        if (S.dups) atomicAdd(counters + CNT_DUPS, (unsigned long long)S.dups);
    }
}

// The result from the staged pairs of group g, at [g * slot, g * slot + nuniq), or for a fallback group from the generic
// path's uniques (k_fallback_place: g_src); the destination of group g starts at uoff[g]
__global__ void k_compact_uniq(const uint64_t *__restrict__ st_hash, const uint32_t *__restrict__ st_cnt,
                               uint32_t slot, const uint32_t *__restrict__ g_nuniq,
                               const uint32_t *__restrict__ uoff, const uint8_t *__restrict__ g_fallback,
                               const uint32_t *__restrict__ g_src, const uint64_t *__restrict__ f_hash,
                               const uint32_t *__restrict__ f_cnt, uint64_t *__restrict__ out_hash,
                               uint32_t *__restrict__ out_cnt) {
    const uint32_t g = blockIdx.x, nu = g_nuniq[g], u0 = uoff[g];
    const bool fb = g_fallback[g] != 0;
    const uint64_t *sh = fb ? f_hash + g_src[g] : st_hash + (uint64_t)g * slot;
    const uint32_t *sc = fb ? f_cnt + g_src[g] : st_cnt + (uint64_t)g * slot;
    for (uint32_t i = threadIdx.x; i < nu; i += blockDim.x) {
        out_hash[u0 + i] = sh[i];
        out_cnt[u0 + i] = sc[i];
    }
}

// The generic path returns the fallback groups' unique pairs as ONE list sorted by hash.  Groups own
// disjoint, increasing hash ranges (bucket = mulhi(hash, Mb) is monotone), so group g's slice is
// [lower_bound(hash >= first hash of bucket bf), lower_bound(hash >= first hash of bucket be)).
__global__ void k_fallback_place(const uint8_t *__restrict__ g_fallback, uint32_t ng, uint32_t g0, uint32_t nbk, uint64_t Mb,
                                 const uint64_t *__restrict__ f_hash, uint64_t fu, uint32_t *__restrict__ g_nuniq,
                                 uint32_t *__restrict__ g_src) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ng || !g_fallback[g]) return;
    auto first_hash_of = [&](uint32_t b) -> uint64_t {  // smallest h with mulhi(h, Mb) >= b
        const unsigned __int128 num = ((unsigned __int128)b << 64) + (Mb - 1);
        return (uint64_t)(num / Mb);
    };
    auto lb = [&](uint64_t v) -> uint64_t {
        uint64_t lo = 0, hi = fu;
        while (lo < hi) { uint64_t mid = (lo + hi) >> 1; if (f_hash[mid] < v) lo = mid + 1; else hi = mid; }
        return lo;
    };
    const uint32_t bf = (g0 + g) * GRP_BPG, be = bf + GRP_BPG;  // the part's group g is group g0 + g of the map
    const uint64_t a = bf == 0 ? 0 : lb(first_hash_of(bf));
    const uint64_t b = be >= nbk ? fu : lb(first_hash_of(be));
    g_src[g] = (uint32_t)a;
    g_nuniq[g] = (uint32_t)(b - a);
}

// slotted events of fallback groups -> compact SoA arrays for the generic path
__global__ void k_gather_fallback(const EventRec *__restrict__ ev, uint32_t slot,
                                  const uint32_t *__restrict__ g_n, const uint8_t *__restrict__ g_fallback,
                                  const uint32_t *__restrict__ foff, uint64_t *__restrict__ hash,
                                  uint64_t *__restrict__ recflag, uint64_t *__restrict__ p0, uint64_t *__restrict__ p1) {
    const uint32_t g = blockIdx.x;
    if (!g_fallback[g]) return;
    const uint64_t e0 = (uint64_t)g * slot;
    const uint32_t n = g_n[g], f0 = foff[g];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const EventRec r = ev[e0 + i];
        hash[f0 + i] = r.hash; recflag[f0 + i] = r.recflag; p0[f0 + i] = r.p0; p1[f0 + i] = r.p1;
    }
}

__global__ void k_fallback_sizes(const uint32_t *__restrict__ g_n, const uint8_t *__restrict__ g_fallback, uint32_t ng,
                                 uint32_t *__restrict__ fsz) {
    uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < ng) fsz[g] = g_fallback[g] ? g_n[g] : 0u;
}

// Accumulates events over one or more seeding batches, then finishes into a syl_sample.
// Nothing in begin() / add() synchronises with the host: the event array is sized up front from the
// expected number of survivors, the seeding kernel appends at a running device counter, and every
// post-pass kernel reads the event count from device memory with grids sized for the capacity.  The ONE
// host synchronisation of a sketch is in finish(); if the events did not fit (homopolymer reads at tiny c)
// finish() reports the true count and the caller redoes the sample with that capacity.
struct SampleBuilder {
    syl_ctx *ctx;
    int k;
    uint64_t c;
    int no_dedup, sem;
    bool paired;             // read pairs (syl_sketch_read_pairs): every event waits for k_events_fix<.., true>
    uint64_t n_reads;        // records: reads, or pairs
    double mean_read_length;
    uint64_t cap = 0;
    // Event array: ng group slots of `slot` events each, then the overflow list of cap events (everything
    // in the overflow list without groups).  A scratch block of the ctx cache.
    DevBuf<EventRec> b_ev;
    DevBuf<uint32_t> b_pend; // indices of events whose pair keys are filled in by k_events_fix
    // Post-pass groups: fixed before the first batch from the expected number of events, so that the
    // seeding kernel can write every event into its group while it flushes them.
    uint64_t expect_bases = 0, expect_reads = 0;
    uint32_t nbk = 0, ng = 0, slot = 0;
    uint64_t Mb = 0;
    // the part of the sample this pass sketches (sample_parts.hpp): hashes [lo, hi), groups [g0, g0 + ng) of the map
    uint64_t lo = 0, hi = 0;
    uint32_t g0 = 0;
    DevBuf<uint32_t> g_cnt;  // events per group
    // ctx->d_counters: CNT_EVENTS (events in the overflow list), CNT_PENDING, CNT_DUPS; add() keeps CNT_PEND_MATE1 and
    // CNT_PEND_MATE2 as snapshots of CNT_PENDING
    unsigned long long *d_count() const { return reinterpret_cast<unsigned long long *>(ctx->d_counters); }
    uint64_t ev_total() const { return (uint64_t)ng * slot + cap; }

    // map: the one-pass group map of the whole sample; part: the hashes this pass keeps (all of them: lo 0, hi thr).
    // grouped: false for SYL_SAMPLE_POSTPASS=sort (no groups, every event takes the generic path).
    int begin(const SampleMap &map, const SamplePart &part, bool grouped, uint64_t cap_override) {
        cudaStream_t st = ctx->stream;
        lo = part.lo;
        hi = part.hi;
        g0 = part.g0;
        if (grouped) {
            static const uint32_t grp_cap = []() { const char *e = getenv("SYL_GROUP_CAP"); int v = e ? atoi(e) : GRP_CAP; return (uint32_t)std::min(std::max(v, 32), GRP_CAP); }();
            slot = grp_cap;
            ng = part.ng;
            nbk = map.nbk;
            Mb = map.Mb;
            SYL_TRY(g_cnt.alloc(ng, st));
            SYL_CUDA(cudaMemsetAsync(g_cnt.p, 0, (size_t)ng * 4, st));
        }
        // with groups cap is the overflow list, almost always empty: 1/16 of the estimate; a sample that
        // needs more (duplicate-heavy, homopolymers) is redone with the exact length
        cap = overflow_cap(part_bases(expect_bases, lo, hi, map.thr), c, grouped);
        if (cap_override) cap = cap_override;
        if (ev_total() >= 0xFFFFFFFEull) { set_error("more than 2^32-2 survivor events in one sample"); return SYL_ERR_ARG; }
        SYL_TRY(b_ev.alloc(ev_total(), st));
        SYL_TRY(b_pend.alloc(ev_total(), st));
        SYL_CUDA(cudaMemsetAsync(ctx->d_counters, 0, 6 * sizeof(uint64_t), st));  // CNT_EVENTS .. CNT_FALLBACK_TOTAL
        return SYL_OK;
    }

    // One batch of records [rec_base, rec_base + nr) (batches may arrive in any order), device resident: m[0] for
    // reads, m[0] and m[1] for read pairs.  Each mate is seeded with the record index as read index; the seeding kernel
    // appends the events (hash, record, pair keys) to the event array.  The pending events are then completed while
    // the batch is resident: reads cut by a tile edge, whose keys come from global memory, and every event of a pair,
    // whose keys need both mates.  CNT_PENDING counts the pending events; CNT_PEND_MATE1 / 2 keep its value from before
    // mate 1 and mate 2, so the batch's pending events are pend[[CNT_PEND_MATE1] .. [CNT_PENDING]) and mate 2's start at
    // [CNT_PEND_MATE2].
    int add(const Mate *m, int n_mates, uint64_t nr, uint64_t rec_base) {
        cudaStream_t st = ctx->stream;
        if (nr == 0) return SYL_OK;
        unsigned long long *dc = d_count();
        for (int i = 0; i < n_mates; i++) {
            SYL_CUDA(cudaMemcpyAsync(dc + (i ? CNT_PEND_MATE2 : CNT_PEND_MATE1), dc + CNT_PENDING, 8, cudaMemcpyDeviceToDevice, st));
            SeedJob job;
            job.d_bases = m[i].bases; job.d_packed = m[i].packed; job.n_bases = m[i].nb; job.d_rec_off = m[i].off;
            job.off_bias = m[i].off_bias; job.n_rec = nr; job.k = k; job.c = c; job.sem = sem; job.with_pos = 0;
            job.d_out = b_ev.p; job.cap = cap; job.emit_events = 1; job.rec_base = rec_base;
            job.no_dedup = paired ? 2 : no_dedup; job.d_pend = b_pend.p;
            job.d_group_cnt = g_cnt.p; job.Mb = Mb; job.nbk = nbk; job.ng = ng; job.slot = slot; job.d_count = dc;
            job.g0 = g0; job.lo = lo; job.hi = hi;
            SYL_TRY(seed_enqueue(ctx, job));
        }
        if (!paired && (no_dedup || !m[0].nb)) return SYL_OK;  // no pending events
        auto fix = paired ? (m[0].packed ? k_events_fix<true, true> : k_events_fix<false, true>)
                          : (m[0].packed ? k_events_fix<true, false> : k_events_fix<false, false>);
        fix<<<ctx->num_sms * 2, EV_THREADS, 0, st>>>(b_ev.p, b_pend.p, dc + CNT_PEND_MATE1, dc + CNT_PEND_MATE2, dc + CNT_PENDING,
                                                     ev_total(), m[0], m[n_mates - 1], rec_base, no_dedup);
        ctx->launches++;
        SYL_CUDA(cudaGetLastError());
        return SYL_OK;
    }

    // Generic path: two stable LSD radix sorts (read index, then hash) + run-length encode +
    // k_dedup.  Handles any segment length in linear time; used for the groups the primary
    // path hands over (and for everything when SYL_SAMPLE_POSTPASS=sort).
    int dedup_sorted(const uint64_t *ev_hash, const uint64_t *ev_recflag, const uint64_t *ev_p0, const uint64_t *ev_p1,
                     uint64_t N, DevBuf<uint64_t> &uniq, DevBuf<uint32_t> &count, uint64_t *U_out, uint64_t *ndup_out) {
        cudaStream_t st = ctx->stream;
        *U_out = 0;
        *ndup_out = 0;
        if (N == 0) return SYL_OK;
        DevBuf<uint32_t> idx_a, idx_b;
        DevBuf<uint64_t> key_a, key_b;
        SYL_TRY(idx_a.alloc(N, st)); SYL_TRY(idx_b.alloc(N, st));
        SYL_TRY(key_a.alloc(N, st)); SYL_TRY(key_b.alloc(N, st));
        k_iota<<<nblk(N, 256), 256, 0, st>>>(idx_a.p, N);
        ctx->launches++;
        const int hash_bits = bits_for(fmh_threshold(c));
        DevBuf<uint8_t> tmp;
        size_t tmp_bytes = 0, t2 = 0;
        uint32_t *ord = idx_a.p;  // final event order
        uint64_t *hs = key_a.p;   // hashes in final order
        if (!no_dedup || paired) {
            const int rec_bits = paired ? bits_for((n_reads << 2) | 3) : bits_for((n_reads << 1) | 1);
            cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ev_recflag, key_b.p, idx_a.p, idx_b.p, N, 0, rec_bits, st);
            cub::DeviceRadixSort::SortPairs(nullptr, t2, key_a.p, key_b.p, idx_b.p, idx_a.p, N, 0, hash_bits, st);
            tmp_bytes = std::max(tmp_bytes, t2);
            SYL_TRY(tmp.alloc(tmp_bytes, st));
            SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, ev_recflag, key_b.p, idx_a.p, idx_b.p, N, 0, rec_bits, st));
            k_gather<uint64_t><<<nblk(N, 256), 256, 0, st>>>(ev_hash, idx_b.p, key_a.p, N);
            SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, key_a.p, key_b.p, idx_b.p, idx_a.p, N, 0, hash_bits, st));
            ctx->launches += 3;
            hs = key_b.p;
            ord = idx_a.p;
        } else {
            cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, ev_hash, key_b.p, N, 0, hash_bits, st);
            SYL_TRY(tmp.alloc(tmp_bytes, st));
            SYL_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tmp_bytes, ev_hash, key_b.p, N, 0, hash_bits, st));
            ctx->launches += 1;
            hs = key_b.p;
        }
        DevBuf<uint64_t> seg_off;
        DevBuf<uint32_t> seg_len;
        SYL_TRY(uniq.alloc(N, st)); SYL_TRY(seg_off.alloc(N + 1, st)); SYL_TRY(seg_len.alloc(N, st));
        uint64_t *d_nruns = ctx->d_counters + CNT_PENDING;
        size_t rle_bytes = 0, scan_bytes = 0;
        cub::DeviceRunLengthEncode::Encode(nullptr, rle_bytes, hs, uniq.p, seg_len.p, d_nruns, N, st);
        cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, seg_len.p, seg_off.p, N, st);
        DevBuf<uint8_t> tmp2;
        SYL_TRY(tmp2.alloc(std::max(rle_bytes, scan_bytes), st));
        size_t tb = std::max(rle_bytes, scan_bytes);
        SYL_CUDA(cub::DeviceRunLengthEncode::Encode(tmp2.p, tb, hs, uniq.p, seg_len.p, d_nruns, N, st));
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_PENDING, d_nruns, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        const uint64_t U = ctx->h_counters[CNT_PENDING];
        ctx->launches += 1;
        SYL_TRY(count.alloc(std::max<uint64_t>(U, 1), st));
        if (no_dedup && !paired) {
            SYL_CUDA(cudaMemcpyAsync(count.p, seg_len.p, U * 4, cudaMemcpyDeviceToDevice, st));
        } else {
            tb = std::max(rle_bytes, scan_bytes);
            SYL_CUDA(cub::DeviceScan::ExclusiveSum(tmp2.p, tb, seg_len.p, seg_off.p, U, st));
            DevBuf<uint64_t> set;
            SYL_TRY(set.alloc(2 * N, st));
            unsigned long long *d_ndup = reinterpret_cast<unsigned long long *>(ctx->d_counters + CNT_DUPS);
            SYL_CUDA(cudaMemsetAsync(d_ndup, 0, 8, st));
            if (paired) k_dedup_paired<<<nblk(U * 32, 128), 128, 0, st>>>(seg_off.p, seg_len.p, U, ord, ev_recflag, ev_p0, ev_p1, no_dedup, set.p, count.p, d_ndup);
            else k_dedup<<<nblk(U, 128), 128, 0, st>>>(seg_off.p, seg_len.p, U, ord, ev_recflag, ev_p0, ev_p1, set.p, count.p, d_ndup);
            ctx->launches += 2;
            SYL_CUDA(cudaGetLastError());
            SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_DUPS, d_ndup, 8, cudaMemcpyDeviceToHost, st));
            SYL_CUDA(cudaStreamSynchronize(st));
            *ndup_out = ctx->h_counters[CNT_DUPS];
        }
        *U_out = U;
        return SYL_OK;
    }

    // need_cap: set when SYL_ERR_CAPACITY is returned (the true number of events)
    int finish(syl_sample **out, uint64_t *need_cap) {
        cudaStream_t st = ctx->stream;
        *need_cap = 0;
        Handle<syl_sample> s = new_handle<syl_sample>(ctx);
        if (!s) return SYL_ERR_OOM;
        s->k = k;
        s->c = c;
        s->mean_read_length = mean_read_length;
        if (n_reads == 0 || expect_bases == 0) { *out = s.release(); return SYL_OK; }
        unsigned long long *dc = d_count();
        EventRec *ev = b_ev.p;
        // ---- primary path: CTA-local grouping / dedup of the group slots (ng, slot, Mb, g_cnt: begin()).
        // The kernels read the group counts from device memory.  k_group_dedup writes each group's sorted uniques into
        // the group's slot of the staging arrays and sums the uniques (and the slotted events of the fallback groups)
        // into the device counters, so one scan of the per-group counts before the sync and one compaction into the
        // exact-size result after it complete the sketch.
        const uint64_t n_slots = (uint64_t)ng * slot;
        DevBuf<uint32_t> st_cnt, g_nuniq, g_n, uoff, fsz, foff, g_src;
        DevBuf<uint64_t> st_hash;
        DevBuf<uint8_t> g_fb;
        if (ng) {
            SYL_TRY(st_hash.alloc(n_slots, st)); SYL_TRY(st_cnt.alloc(n_slots, st));  // in-kernel uniques <= slotted events
            SYL_TRY(g_nuniq.alloc(ng, st)); SYL_TRY(g_n.alloc(ng, st)); SYL_TRY(g_fb.alloc(ng, st));
            SYL_TRY(uoff.alloc((uint64_t)ng + 1, st)); SYL_TRY(g_src.alloc(ng, st));
            auto group_dedup = paired ? k_group_dedup<true> : k_group_dedup<false>;
            const int smem = paired ? (int)sizeof(GroupSmem<true>) : (int)sizeof(GroupSmem<false>);
            SYL_CUDA(cudaFuncSetAttribute(group_dedup, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            {
                KernelTimer kt(ctx, SYL_KERNEL_GROUP_DEDUP);
                group_dedup<<<ng, GRP_THREADS, smem, st>>>(ev, g_cnt.p, slot, Mb, nbk, g0, no_dedup, st_hash.p, st_cnt.p,
                                                            g_nuniq.p, g_n.p, g_fb.p, dc);
            }
            k_scan_u32<<<1, 1024, 0, st>>>(g_nuniq.p, ng, uoff.p);
            ctx->launches += 2;
            SYL_CUDA(cudaGetLastError());
        }
        // CNT_EVENTS, CNT_PENDING, CNT_DUPS, CNT_PEND_MATE1, CNT_UNIQ_TOTAL, CNT_FALLBACK_TOTAL (all cleared in begin())
        static_assert(CNT_UNIQ_TOTAL == 4 && CNT_FALLBACK_TOTAL == 5, "one copy of slots 0 .. 5");
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters, dc, 6 * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));  // the one synchronisation of a sketch
        const uint64_t N_ovf = ctx->h_counters[CNT_EVENTS];
        if (N_ovf > cap) { *need_cap = N_ovf; return SYL_ERR_CAPACITY; }
        // the overflow list holds only events of groups past their slot, all of which are fallback groups (without
        // groups: every event)
        const uint64_t U1 = ng ? ctx->h_counters[CNT_UNIQ_TOTAL] : 0;
        const uint64_t NF_slots = ng ? ctx->h_counters[CNT_FALLBACK_TOTAL] : 0;
        const uint64_t NF = NF_slots + N_ovf;
        uint64_t ndup = ctx->h_counters[CNT_DUPS];
        if (debug_timing()) fprintf(stderr, "[sample post-pass] groups %u of %u slots, overflow list %llu (cap %llu): in-kernel uniques %llu, events handed to the generic path %llu (%.2f %% of the slotted events)\n",
                         ng, slot, (unsigned long long)N_ovf, (unsigned long long)cap, (unsigned long long)U1, (unsigned long long)NF,
                         n_slots ? 100.0 * (double)NF_slots / (double)n_slots : 0.);
        // the generic path: fallback groups (heavy-hitter k-mers, duplicate-heavy replays) and the overflow list
        DevBuf<uint64_t> fh, f_rf, f_p0, f_p1, f_uq;
        DevBuf<uint32_t> f_ct;
        uint64_t U2 = 0;
        if (NF) {
            uint64_t nd2 = 0;
            SYL_TRY(fh.alloc(NF, st)); SYL_TRY(f_rf.alloc(NF, st)); SYL_TRY(f_p0.alloc(NF, st)); SYL_TRY(f_p1.alloc(NF, st));
            if (NF_slots) {  // the fallback groups' slotted events, compacted in group order
                SYL_TRY(fsz.alloc(ng, st)); SYL_TRY(foff.alloc((uint64_t)ng + 1, st));
                k_fallback_sizes<<<nblk(ng, 256), 256, 0, st>>>(g_n.p, g_fb.p, ng, fsz.p);
                k_scan_u32<<<1, 1024, 0, st>>>(fsz.p, ng, foff.p);
                k_gather_fallback<<<ng, 256, 0, st>>>(ev, slot, g_n.p, g_fb.p, foff.p, fh.p, f_rf.p, f_p0.p, f_p1.p);
                ctx->launches += 3;
            }
            if (N_ovf) {
                k_unpack_events<<<nblk(N_ovf, 256), 256, 0, st>>>(ev + n_slots, N_ovf, fh.p + NF_slots, f_rf.p + NF_slots,
                                                                  f_p0.p + NF_slots, f_p1.p + NF_slots);
                ctx->launches++;
            }
            SYL_TRY(dedup_sorted(fh.p, f_rf.p, f_p0.p, f_p1.p, NF, f_uq, f_ct, &U2, &nd2));
            ndup += nd2;
        }
        // exact-size result arrays; the copies are ordered on the ctx stream like every later use of the handle
        const uint64_t U = U1 + U2;
        SYL_TRY(hblock_alloc(ctx, (void **)&s->hash, std::max<uint64_t>(U, 1) * 8));
        SYL_TRY(hblock_alloc(ctx, (void **)&s->count, std::max<uint64_t>(U, 1) * 4));
        if (ng) {
            if (U2) {  // slot the generic path's pairs into the fallback groups' positions
                k_fallback_place<<<nblk(ng, 128), 128, 0, st>>>(g_fb.p, ng, g0, nbk, Mb, f_uq.p, U2, g_nuniq.p, g_src.p);
                k_scan_u32<<<1, 1024, 0, st>>>(g_nuniq.p, ng, uoff.p);
                ctx->launches += 2;
            }
            k_compact_uniq<<<ng, 128, 0, st>>>(st_hash.p, st_cnt.p, slot, g_nuniq.p, uoff.p, g_fb.p, g_src.p, f_uq.p, f_ct.p,
                                                s->hash, s->count);
            ctx->launches++;
            SYL_CUDA(cudaGetLastError());
        } else if (U) {  // without groups: the generic path's uniques
            SYL_CUDA(cudaMemcpyAsync(s->hash, f_uq.p, U * 8, cudaMemcpyDeviceToDevice, st));
            SYL_CUDA(cudaMemcpyAsync(s->count, f_ct.p, U * 4, cudaMemcpyDeviceToDevice, st));
        }
        if (NF) SYL_CUDA(cudaStreamSynchronize(st));  // f_uq / f_ct go out of scope
        s->n = U;
        s->num_dup_removed = ndup;
        *out = s.release();
        return SYL_OK;
    }
};

}  // namespace syl

namespace syl {

// The chunks of host ASCII reads or pairs (ingest.hpp): records [r0, r1), at most the chunk size of the mode in bases
static void plan_read_chunks(const Mate *m, int n_mates, uint64_t n_reads, bool ascii_only, std::vector<Chunk> &chunks) {
    if (ascii_only) plan_chunks(m, n_mates, n_reads, ingest_chunk(ING_ASCII_CHUNK), n_reads, chunks);
    else plan_chunks(m, n_mates, n_reads, ingest_chunk(ING_CHUNK), ING_MAXREC / n_mates, chunks);
}

// Bytes of the rings the ctx holds now (syl_ctx_ingest_ring_bytes)
static uint64_t ring_bytes_now(const syl_ctx *ctx) {
    uint64_t d = 0;
    syl_ctx_ingest_ring_bytes(ctx, &d, nullptr);
    return d;
}

// The hash-range parts of a sample (sample_parts.hpp) within the ctx's budget (syl_ctx_set_sample_memory; 0: the free
// device memory now, plus the ctx's cached free blocks and rings, which the call reuses).  The fixed bytes are the
// staging rings for host ASCII, or host 2-bit input staged whole.  SYL_SAMPLE_PARTS=N (read per call) forces N parts.
// Nothing is allocated here: a budget the plan cannot meet fails before the call touches the device.
static int plan_parts(syl_ctx *ctx, int mem, bool packed, bool ascii_only, const Mate *m, int n_mates, uint64_t n_reads,
                      uint64_t bases, int k, uint64_t c, bool grouped, SamplePlan &plan) {
    uint64_t fixed = 0;
    for (int i = 0; i < n_mates; i++) fixed += (seed_cta_tiles(m[i].nb) + 1) * 4 + 256;  // the seeding kernel's tile table
    if (mem == SYL_MEM_HOST && packed)
        for (int i = 0; i < n_mates; i++) fixed += ((m[i].nb + 15) / 16 + 16) * 4 + (n_reads + 9) * 8;
    else if (mem == SYL_MEM_HOST) {
        std::vector<Chunk> chunks;
        if (n_reads) plan_read_chunks(m, n_mates, n_reads, ascii_only, chunks);
        fixed += ring_bytes_after(ctx, chunks, n_mates, ascii_only);
    }
    uint32_t forced = 0;
    if (const char *e = getenv("SYL_SAMPLE_PARTS")) forced = (uint32_t)std::max(0, atoi(e));
    uint64_t budget = ctx->sample_budget;
    if (!budget) {
        uint64_t held = ring_bytes_now(ctx);
        for (const auto &b : ctx->free_blocks) held += b.second;
        // cudaMemGetInfo costs about as much as a small sketch's post-pass: a sample whose one pass needs less than
        // half of the free memory this ctx last saw takes one pass without asking again
        if (!forced && plan_sample_parts(bases, n_reads, n_mates, k, c, grouped, UINT64_MAX, fixed, 0, plan) == PLAN_OK &&
            plan.parts.size() == 1 && plan.need <= held + ctx->free_seen / 2)
            return SYL_OK;
        size_t free_b = 0, total_b = 0;
        SYL_CUDA(cudaMemGetInfo(&free_b, &total_b));
        ctx->free_seen = free_b;
        budget = free_b + held;
    }
    switch (plan_sample_parts(bases, n_reads, n_mates, k, c, grouped, budget, fixed, forced, plan)) {
        case PLAN_OK: return SYL_OK;
        case PLAN_TOO_MANY_EVENTS: set_error("more than 2^32-2 survivor events in one sample part"); return SYL_ERR_ARG;
        default:
            set_error("sketching this sample needs " + std::to_string(plan.need) + " bytes of device memory in " +
                      std::to_string(SAMPLE_MAX_PARTS) + " parts, the budget is " + std::to_string(budget) + " bytes");
            return SYL_ERR_OOM;
    }
}

// A sample of n_reads records: reads (n_mates 1), or read pairs (n_mates 2: mate i of pair p is record p of m[i]).
// packed: every mate is 2-bit words, else ASCII; mem: where all of it lives.  Device input is used in place, host
// 2-bit words (a quarter of the bytes) are staged whole once per call, host ASCII goes through feed_host in chunks.
// A sample whose post-pass does not fit the ctx's budget is sketched in parts, one hash range per pass over the input
// (host ASCII is fed again for every part); each part's sketch waits in host memory, and the parts, in range order,
// are the sketch.  A part with more events than estimated is redone (host ASCII: fed again) with the exact event capacity.
static int sketch_reads_impl(syl_ctx *ctx, int mem, bool packed, const Mate *m, int n_mates, uint64_t n_reads, int k,
                             uint64_t c, int no_dedup, int sem, syl_sample **out) {
    bool null_arg = !ctx || !out;
    for (int i = 0; i < n_mates; i++) null_arg = null_arg || (!m[i].bases && !m[i].packed && m[i].nb) || !m[i].off;
    if (null_arg) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (c == 0) { set_error("c must be >= 1"); return SYL_ERR_ARG; }
    if (mem != SYL_MEM_HOST && mem != SYL_MEM_DEVICE) { set_error("bad mem"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_ENTER(ctx);
    const bool fed = mem == SYL_MEM_HOST && !packed;
    const bool host_ascii = host_ingest_ascii();
    const char *pp = getenv("SYL_SAMPLE_POSTPASS");  // per call; "sort": no groups, every event takes the generic path
    const bool grouped = !(pp && std::string(pp) == "sort");
    uint64_t expect_bases = 0;
    for (int i = 0; i < n_mates; i++) expect_bases += m[i].nb;
    SamplePlan plan;
    SYL_TRY(plan_parts(ctx, mem, packed, host_ascii, m, n_mates, n_reads, expect_bases, k, c, grouped, plan));
    const size_t P = plan.parts.size();
    ctx->sample_parts = (uint32_t)P;
    if (P > 1) SYL_TRY(cache_trim(ctx));  // every part's pass is allocated to its own size, not next to cached blocks
    Mate dm[2] = {};  // the mates on the device, unless fed
    Staged<uint32_t> sp[2];
    Staged<uint64_t> so[2];
    uint64_t staged_bytes = 0;
    for (int i = 0; i < n_mates; i++) {
        if (fed) continue;
        dm[i] = m[i];
        if (packed) { SYL_TRY(sp[i].init(ctx, mem, m[i].packed, (m[i].nb + 15) / 16)); dm[i].packed = sp[i].p; }
        SYL_TRY(so[i].init(ctx, mem, m[i].off, n_reads + 1));
        dm[i].off = so[i].p;
        if (mem == SYL_MEM_HOST) staged_bytes += (m[i].nb + 15) / 16 * 4 + (n_reads + 1) * 8;
    }
    // the mean length of mate 1 (for pairs src/sketch.rs:824-826)
    const double mean_read_length = n_reads ? (double)m[0].nb / (double)n_reads : 0.;
    auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    uint64_t h2d = staged_bytes, n_packed = 0, n_ascii = 0;  // host ingest of the parts so far
    std::vector<uint64_t> all_hash;  // the sketches of the parts so far (P > 1)
    std::vector<uint32_t> all_cnt;
    uint64_t ndup = 0;
    for (size_t p = 0; p < P; p++) {
        const SamplePart &part = plan.parts[p];
        if (P > 1 && part.lo == part.hi) continue;  // a range no hash falls in
        syl_sample *ps = nullptr;
        uint64_t cap_override = 0;
        int rc = SYL_ERR_CAPACITY;
        for (int attempt = 0; attempt < 3 && rc == SYL_ERR_CAPACITY; attempt++) {
            SampleBuilder b{ctx, k, c, no_dedup, sem, n_mates == 2, n_reads, mean_read_length};
            b.expect_bases = expect_bases;
            b.expect_reads = n_mates * n_reads;
            if (mem == SYL_MEM_HOST) {
                ctx->ingest_h2d_bytes = h2d;
                ctx->ingest_chunks_packed = n_packed;
                ctx->ingest_chunks_ascii = n_ascii;
            }
            SYL_TRY(b.begin(plan.map, part, grouped, cap_override));
            const double t0 = now();
            rc = SYL_OK;
            if (!fed) rc = b.add(dm, n_mates, n_reads, 0);
            else if (n_reads && expect_bases) {
                std::vector<Chunk> chunks;
                plan_read_chunks(m, n_mates, n_reads, host_ascii, chunks);
                rc = feed_host(ctx, m, n_mates, chunks, host_ascii, [&](const Mate *dm, size_t ci) {
                    return b.add(dm, n_mates, chunks[ci].r1 - chunks[ci].r0, chunks[ci].r0);
                });
            }
            if (rc != SYL_OK) return rc;
            const double t1 = now();
            uint64_t need = 0;
            rc = b.finish(&ps, &need);
            if (debug_timing()) fprintf(stderr, "[%s] feed %.2f ms, finish %.2f ms (attempt %d)%s\n",
                             n_mates == 2 ? "syl_sketch_read_pairs" : "syl_sketch_reads", t1 - t0, now() - t1, attempt,
                             P > 1 ? (", part " + std::to_string(p + 1) + "/" + std::to_string(P)).c_str() : "");
            if (rc == SYL_ERR_CAPACITY) cap_override = need + 16;  // more events than estimated: redo with the exact size
        }
        if (rc == SYL_ERR_CAPACITY) { set_error("event capacity retry failed"); return SYL_ERR_CAPACITY; }
        SYL_TRY(rc);
        if (P == 1) { *out = ps; return SYL_OK; }
        Handle<syl_sample> hs(ps);
        h2d = ctx->ingest_h2d_bytes;
        n_packed = ctx->ingest_chunks_packed;
        n_ascii = ctx->ingest_chunks_ascii;
        const size_t u0 = all_hash.size();
        all_hash.resize(u0 + hs->n);
        all_cnt.resize(u0 + hs->n);
        SYL_TRY(syl_sample_download(ctx, hs.get(), all_hash.data() + u0, all_cnt.data() + u0));
        ndup += hs->num_dup_removed;
        hs.reset();
        SYL_TRY(cache_trim(ctx));
    }
    // the parts' sketches, in range order, into the exact-size handle
    Handle<syl_sample> s = new_handle<syl_sample>(ctx);
    if (!s) return SYL_ERR_OOM;
    const uint64_t U = all_hash.size();
    s->k = k;
    s->c = c;
    s->mean_read_length = mean_read_length;
    s->num_dup_removed = ndup;
    s->n = U;
    SYL_TRY(hblock_alloc(ctx, (void **)&s->hash, std::max<uint64_t>(U, 1) * 8));
    SYL_TRY(hblock_alloc(ctx, (void **)&s->count, std::max<uint64_t>(U, 1) * 4));
    if (U) {
        SYL_CUDA(cudaMemcpyAsync(s->hash, all_hash.data(), U * 8, cudaMemcpyHostToDevice, ctx->stream));
        SYL_CUDA(cudaMemcpyAsync(s->count, all_cnt.data(), U * 4, cudaMemcpyHostToDevice, ctx->stream));
        SYL_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    *out = s.release();
    return SYL_OK;
}

}  // namespace syl

using namespace syl;

extern "C" {

int syl_sketch_reads(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                     const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup,
                     int sem, syl_sample **out) {
    const Mate m[1] = {{bases, nullptr, n_bases, rec_off, 0}};
    return sketch_reads_impl(ctx, mem, false, m, 1, n_reads, k, c, no_dedup, sem, out);
}

int syl_sketch_reads_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                             const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup,
                             int sem, syl_sample **out) {
    const Mate m[1] = {{nullptr, packed, n_bases, rec_off, 0}};
    return sketch_reads_impl(ctx, mem, true, m, 1, n_reads, k, c, no_dedup, sem, out);
}

int syl_sketch_read_pairs(syl_ctx *ctx, int mem, const uint8_t *bases1, uint64_t n_bases1, const uint64_t *rec_off1,
                          const uint8_t *bases2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                          int k, uint64_t c, int no_dedup, int sem, syl_sample **out) {
    const Mate m[2] = {{bases1, nullptr, n_bases1, rec_off1, 0}, {bases2, nullptr, n_bases2, rec_off2, 0}};
    return sketch_reads_impl(ctx, mem, false, m, 2, n_pairs, k, c, no_dedup, sem, out);
}

int syl_sketch_read_pairs_packed2(syl_ctx *ctx, int mem, const uint32_t *packed1, uint64_t n_bases1, const uint64_t *rec_off1,
                                  const uint32_t *packed2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                                  int k, uint64_t c, int no_dedup, int sem, syl_sample **out) {
    const Mate m[2] = {{nullptr, packed1, n_bases1, rec_off1, 0}, {nullptr, packed2, n_bases2, rec_off2, 0}};
    return sketch_reads_impl(ctx, mem, true, m, 2, n_pairs, k, c, no_dedup, sem, out);
}

int syl_pack_threads(void) { return default_pack_threads(); }

int syl_ctx_set_sample_memory(syl_ctx *ctx, uint64_t max_bytes) {
    if (!ctx) { set_error("NULL argument"); return SYL_ERR_ARG; }
    ctx->sample_budget = max_bytes;
    return SYL_OK;
}

int syl_ctx_sample_memory(syl_ctx *ctx, uint64_t *max_bytes, uint64_t *free_bytes) {
    if (!ctx) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (max_bytes) *max_bytes = ctx->sample_budget;
    if (free_bytes) {
        SYL_ENTER(ctx);
        size_t free_b = 0, total_b = 0;
        SYL_CUDA(cudaMemGetInfo(&free_b, &total_b));
        *free_bytes = free_b;
    }
    return SYL_OK;
}

int syl_ctx_sample_parts(const syl_ctx *ctx, uint32_t *parts) {
    if (!ctx || !parts) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *parts = ctx->sample_parts;
    return SYL_OK;
}

int syl_pack2(const uint8_t *bases, uint64_t n_bases, uint32_t *words, int n_threads) {
    if ((!bases && n_bases) || (!words && n_bases)) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (n_threads <= 0) n_threads = default_pack_threads();
    const uint64_t slice = 1ull << 20;  // bases per task (multiple of 16)
    const uint64_t n_tasks = (n_bases + slice - 1) / slice;
    n_threads = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)n_threads, n_tasks));
    std::atomic<uint64_t> next(0);
    auto work = [&]() {
        for (;;) {
            const uint64_t t = next.fetch_add(1);
            if (t >= n_tasks) break;
            const uint64_t o = t * slice;
            pack2_range(bases + o, std::min(slice, n_bases - o), words + o / 16);
        }
    };
    std::vector<std::thread> th;
    for (int i = 1; i < n_threads; i++) th.emplace_back(work);
    work();
    for (auto &t : th) t.join();
    return SYL_OK;
}

int syl_sample_upload(syl_ctx *ctx, int mem, const uint64_t *hash, const uint32_t *count,
                      uint64_t n, int k, uint64_t c, syl_sample **out) {
    if (!ctx || !out || (n && (!hash || !count))) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_ENTER(ctx);
    cudaStream_t st = ctx->stream;
    Handle<syl_sample> s = new_handle<syl_sample>(ctx);
    if (!s) return SYL_ERR_OOM;
    s->k = k; s->c = c; s->n = n;
    SYL_TRY(hblock_alloc(ctx, (void **)&s->hash, std::max<uint64_t>(n, 1) * 8));
    SYL_TRY(hblock_alloc(ctx, (void **)&s->count, std::max<uint64_t>(n, 1) * 4));
    if (n) {
        DevBuf<uint64_t> kin;
        DevBuf<uint32_t> vin;
        SYL_TRY(kin.alloc(n, st)); SYL_TRY(vin.alloc(n, st));
        cudaMemcpyKind kind = mem == SYL_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        SYL_CUDA(cudaMemcpyAsync(kin.p, hash, n * 8, kind, st));
        SYL_CUDA(cudaMemcpyAsync(vin.p, count, n * 4, kind, st));
        size_t tb = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tb, kin.p, s->hash, vin.p, s->count, n, 0, 64, st);
        DevBuf<uint8_t> tmp;
        SYL_TRY(tmp.alloc(tb, st));
        SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, kin.p, s->hash, vin.p, s->count, n, 0, 64, st));
        ctx->launches += 8;
        SYL_CUDA(cudaStreamSynchronize(st));
    }
    *out = s.release();
    return SYL_OK;
}

uint64_t syl_sample_size(const syl_sample *s) { return s ? s->n : 0; }
double syl_sample_mean_read_length(const syl_sample *s) { return s ? s->mean_read_length : 0.; }
uint64_t syl_sample_num_dup_removed(const syl_sample *s) { return s ? s->num_dup_removed : 0; }
void syl_sample_set_mean_read_length(syl_sample *s, double v) { if (s) s->mean_read_length = v; }

int syl_sample_download(syl_ctx *ctx, const syl_sample *s, uint64_t *hash, uint32_t *count) {
    if (!ctx || !s) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    if (s->n && hash) SYL_CUDA(cudaMemcpyAsync(hash, s->hash, s->n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (s->n && count) SYL_CUDA(cudaMemcpyAsync(count, s->count, s->n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    SYL_CUDA(cudaStreamSynchronize(ctx->stream));
    return SYL_OK;
}

int syl_sample_device_ptrs(const syl_sample *s, const uint64_t **hash, const uint32_t **count) {
    if (!s) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (hash) *hash = s->hash;
    if (count) *count = s->count;
    return SYL_OK;
}

void syl_sample_free(syl_sample *s) {
    if (!s) return;
    cudaSetDevice(s->device);
    hblock_free(s->owner, s->hash);   // back into the owning ctx's block cache
    hblock_free(s->owner, s->count);
    delete s;
}

}  // extern "C"
