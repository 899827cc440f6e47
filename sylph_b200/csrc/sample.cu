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
#include <cub/cub.cuh>

#include <chrono>
#include <cstdlib>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "common.cuh"
#include "host_pack.hpp"
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

// events pend[*p_begin .. *p_end) (indices into ev) belong to the batch (bases | packed, rec_off, off_bias)
template <bool PACKED>
__global__ void __launch_bounds__(EV_THREADS)
k_events_fix(EventRec *__restrict__ ev, const uint32_t *__restrict__ pend, const unsigned long long *__restrict__ p_begin,
             const unsigned long long *__restrict__ p_end, uint64_t ev_cap, const uint8_t *__restrict__ bases,
             const uint32_t *__restrict__ packed, uint64_t n_words, const uint64_t *__restrict__ rec_off, uint64_t off_bias,
             uint64_t rec_base) {
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
    const uint64_t i0 = *p_begin, i1 = *p_end;
    for (uint64_t i = i0 + (uint64_t)blockIdx.x * EV_THREADS + threadIdx.x; i < i1; i += (uint64_t)gridDim.x * EV_THREADS) {
        const uint32_t ei = pend[i];
        if (ei >= ev_cap) continue;
        EventRec *e = ev + ei;
        const uint64_t rf = e->recflag & ~EV_PENDING;
        const uint64_t rec = (rf >> 1) - rec_base;
        const uint64_t a = rec_off[rec] - off_bias;
        const uint64_t L = rec_off[rec + 1] - off_bias - a;
        uint32_t f, g, r, t;
        if (!PACKED) {
            uint32_t x[8];
            load32_unaligned(bases + a, x);
            f = pack16(x, 0x6420, lut); g = pack16(x, 0x7531, lut);
            load32_unaligned(bases + a + L / 2, x);
            r = pack16(x, 0x6420, lut); t = pack16(x, 0x7531, lut);
        } else {
            const uint64_t x = packed64(packed, n_words, a), y = packed64(packed, n_words, a + L / 2);
            f = even_fields(x); g = even_fields(x << 2);
            r = even_fields(y); t = even_fields(y << 2);
        }
        e->recflag = rf;
        e->p0 = ((uint64_t)f << 32) | r;  // doublepairs.0 = [kmer_f, kmer_r]
        e->p1 = ((uint64_t)g << 32) | t;  // doublepairs.1 = [kmer_g, kmer_t]
    }
}

// Read pairs (src/sketch.rs:658-688 pair_kmer): the two keys come from the first 32 bases of BOTH mates; every event of
// the pair carries them.  Events arrive with recflag = pair << 1 | EV_PENDING; the result is
// recflag = pair << 2 | mate << 1 | NO_PAIR (a mate shorter than 33 bp, or --no-dedup).
// ASCII input: bases1 / bases2; 2-bit input: packed1 / packed2 of n_words1 / n_words2 words.
template <bool PACKED>
__global__ void __launch_bounds__(EV_THREADS)
k_events_fix_paired(EventRec *__restrict__ ev, const uint32_t *__restrict__ pend, const unsigned long long *__restrict__ p_begin,
                    const unsigned long long *__restrict__ p_end, uint64_t ev_cap, const uint8_t *__restrict__ bases1,
                    const uint32_t *__restrict__ packed1, uint64_t n_words1, const uint64_t *__restrict__ off1,
                    const uint8_t *__restrict__ bases2, const uint32_t *__restrict__ packed2, uint64_t n_words2,
                    const uint64_t *__restrict__ off2, uint64_t mate, int no_dedup) {
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
    const uint64_t i0 = *p_begin, i1 = *p_end;
    for (uint64_t i = i0 + (uint64_t)blockIdx.x * EV_THREADS + threadIdx.x; i < i1; i += (uint64_t)gridDim.x * EV_THREADS) {
        const uint32_t ei = pend[i];
        if (ei >= ev_cap) continue;
        EventRec *e = ev + ei;
        const uint64_t pair = (e->recflag & ~EV_PENDING) >> 1;
        const uint64_t a1 = off1[pair], a2 = off2[pair];
        const uint64_t L1 = off1[pair + 1] - a1, L2 = off2[pair + 1] - a2;
        const bool has = !no_dedup && L1 >= 33 && L2 >= 33;  // 2 * 16 + 1 (:660)
        uint64_t p0 = 0, p1 = 0;
        if (has) {
            uint32_t f, g, r, t;
            if (!PACKED) {
                uint32_t x[8];
                load32_unaligned(bases1 + a1, x);
                f = pack16(x, 0x6420, lut); g = pack16(x, 0x7531, lut);
                load32_unaligned(bases2 + a2, x);
                r = pack16(x, 0x6420, lut); t = pack16(x, 0x7531, lut);
            } else {
                const uint64_t x = packed64(packed1, n_words1, a1), y = packed64(packed2, n_words2, a2);
                f = even_fields(x); g = even_fields(x << 2);
                r = even_fields(y); t = even_fields(y << 2);
            }
            p0 = ((uint64_t)f << 32) | r;  // ([kmer_f, kmer_r], [kmer_g, kmer_t]) (:685)
            p1 = ((uint64_t)g << 32) | t;
        }
        e->recflag = (pair << 2) | (mate << 1) | (has ? 0ull : NO_PAIR);
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

__global__ void k_off32_to_64(const uint32_t *__restrict__ in, uint64_t n, uint64_t *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
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

__global__ void k_copy_len(const uint32_t *__restrict__ len, uint32_t *__restrict__ count, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) count[i] = len[i];
}


// ------------------------------------------------------------------------------------------------
// Post-pass, primary path: MSD bucket partition + CTA-local grouping + fused run-length / dedup.
//   the seeding kernel's flush (GroupOut, seed_kernel.cuh) : writes every event into the slot of its
//       group g = bucket / GRP_BPG, bucket = min(mulhi(hash, Mb), nbk - 1) (monotone in the hash, uniform
//       because hashes are uniform below thr); the groups are fixed in begin() at ~GRP_T expected events
//   k_group_dedup : one CTA per group (<= slot events) groups the events by k-mer in shared memory
//       and replays dup_removal_lsh_full_exact per k-mer
//   k_compact_uniq : staged (hash,count) pairs -> dense arrays; buckets are monotone in the hash
//       and every group is sorted, so the result is globally sorted without a merge.
// Groups that do not fit (heavy-hitter k-mers: more events than the slot, the rest in the overflow list)
// or whose dedup set outgrows the per-thread buffer are handed to the generic radix-sort path below and
// merged at the end.
constexpr int GRP_THREADS = 256;
constexpr int GRP_CAP = 1024;   // most events one CTA handles in shared memory (= slot per group)
constexpr int GRP_T = 640;      // expected events per group: room in the slot for the spread of duplicate-heavy k-mers

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
constexpr int GRP_SLOTS = 2048;  // table slots (load factor <= 0.5)
constexpr int GRP_SELECT_STEPS = 64;  // selection steps before a duplicate-heavy k-mer goes to the generic path

struct GroupSmem {
    unsigned long long ht[GRP_SLOTS];  // 16 KB  hash per slot
    uint64_t rf[GRP_CAP];              //  8 KB  recflag per event        | after the replay: unique hashes
    uint64_t p0[GRP_CAP];              //  8 KB  first pair key per event | after the replay: unique counts (u32)
    uint64_t p1[GRP_CAP];              //  8 KB  second pair key per event
    uint16_t scnt[GRP_SLOTS];          //  4 KB  events per slot, then fill cursor, then the k-mer's count
    uint16_t soff[GRP_SLOTS + 2];      //  4 KB  exclusive scan of scnt
    uint16_t ev_slot[GRP_CAP];         //  2 KB  slot per event | after the member fill: 2 x GRP_BPG bucket counters / offsets
    uint16_t member[GRP_CAP];          //  2 KB  event indices grouped by slot
    uint16_t occ[GRP_CAP];             //  2 KB  occupied slots, compacted
    uint32_t wtot[GRP_THREADS / 32], wocc[GRP_THREADS / 32];
    uint32_t overflow, dups, nlong;
    uint16_t longs[GRP_CAP / 2];      //  1 KB  slots of k-mers that need the warp-cooperative replay
};

__global__ void __launch_bounds__(GRP_THREADS)
k_group_dedup(const EventRec *__restrict__ ev, const uint32_t *__restrict__ g_cnt, uint32_t slot, uint64_t Mb, uint32_t nbk,
              int no_dedup, uint64_t *__restrict__ st_hash, uint32_t *__restrict__ st_cnt,
              uint32_t *__restrict__ g_nuniq, uint32_t *__restrict__ g_n,
              uint8_t *__restrict__ g_fallback, unsigned long long *__restrict__ n_dup) {
    extern __shared__ __align__(16) uint8_t grp_smem_raw[];
    GroupSmem &S = *reinterpret_cast<GroupSmem *>(grp_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t g = blockIdx.x;
    if (tid == 0) {
        S.overflow = 0;
        S.dups = 0;
        S.nlong = 0;
    }
    const uint32_t e0 = g * slot, bf = g * GRP_BPG;
    const uint32_t n_all = g_cnt[g], n = min(n_all, slot);  // events past the slot are in the overflow list
    if (tid == 0) { g_n[g] = n; g_nuniq[g] = 0; g_fallback[g] = n_all > slot; }
    if (n == 0 || n_all > slot) return;
    for (int i = tid; i < GRP_SLOTS; i += GRP_THREADS) { S.ht[i] = 0xFFFFFFFFFFFFFFFFull; S.scnt[i] = 0; }
    __syncthreads();
    // (1) stage the events, group equal hashes: slot per event, events per slot
    for (uint32_t i = tid; i < n; i += GRP_THREADS) {
        const uint4 *src = reinterpret_cast<const uint4 *>(ev + e0 + i);
        const uint4 a = __ldcs(src), b = __ldcs(src + 1);  // read once
        const unsigned long long h = ((unsigned long long)a.y << 32) | a.x;
        S.rf[i] = ((uint64_t)a.w << 32) | a.z;
        S.p0[i] = ((uint64_t)b.y << 32) | b.x;
        S.p1[i] = ((uint64_t)b.w << 32) | b.z;
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
        if (no_dedup || len == 1) {
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
                const uint64_t ka = S.p0[m], kb = S.p1[m];
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
            const uint64_t ka = S.p0[bm], kb = S.p1[bm];
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
    if (S.overflow) { if (tid == 0) g_fallback[g] = 1; return; }
    // (3) output order: lb_cnt holds the k-mers per bucket (counted in (2)).
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
    if (tid == 0) { g_nuniq[g] = nu; if (S.dups) atomicAdd(n_dup, (unsigned long long)S.dups); }
}

// staged pairs of group g live at [g * slot, g * slot + nuniq); dense destination starts at uoff[g]
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
__global__ void k_fallback_place(const uint8_t *__restrict__ g_fallback, uint32_t ng, uint32_t nbk, uint64_t Mb,
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
    const uint32_t bf = g * GRP_BPG, be = bf + GRP_BPG;
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

static inline unsigned nblk(uint64_t n, int bs) { return (unsigned)((n + bs - 1) / bs); }

static inline int bits_for(uint64_t maxval) {
    int b = 1;
    while (b < 64 && (maxval >> b)) b++;
    return b;
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
    uint64_t n_reads = 0, n_bases = 0, cap = 0;
    bool paired = false;     // read pairs (syl_sketch_read_pairs): events wait for k_events_fix_paired, generic post-pass only
    bool generic_postpass() const {
        static const bool env_sort = []() { const char *e = getenv("SYL_SAMPLE_POSTPASS"); return e && std::string(e) == "sort"; }();
        return env_sort || paired;
    }
    // Event array: ng group slots of `slot` events each, then the overflow list of cap events (everything
    // in the overflow list without groups).  A scratch block of the ctx cache.
    DevBuf<EventRec> b_ev;
    DevBuf<uint32_t> b_pend; // indices of events whose pair keys are filled in by k_events_fix
    // Post-pass groups: fixed before the first batch from the expected number of events, so that the
    // seeding kernel can write every event into its group while it flushes them.
    uint64_t expect_bases = 0, expect_reads = 0;
    uint32_t nbk = 0, ng = 0, slot = 0;
    uint64_t Mb = 0;
    DevBuf<uint32_t> g_cnt;  // events per group
    // ctx->d_counters slots: [0] events in the overflow list, [1] pending events, [2] duplicates removed, [3] pending snapshot
    unsigned long long *d_count() const { return reinterpret_cast<unsigned long long *>(ctx->d_counters); }
    uint64_t ev_total() const { return (uint64_t)ng * slot + cap; }

    int begin(uint64_t cap_override) {
        cudaStream_t st = ctx->stream;
        const uint64_t win = expect_bases > expect_reads * (uint64_t)(k - 1) ? expect_bases - expect_reads * (uint64_t)(k - 1) : 0;
        const uint64_t n_exp = win / c;
        if (!generic_postpass()) {
            static const uint32_t grp_cap = []() { const char *e = getenv("SYL_GROUP_CAP"); int v = e ? atoi(e) : GRP_CAP; return (uint32_t)std::min(std::max(v, 32), GRP_CAP); }();
            slot = grp_cap;
            const uint64_t g = n_exp / GRP_T + 1;
            if (g * GRP_BPG >= 0xFFFFFFFFull) { set_error("more than 2^32-2 survivor events in one sample"); return SYL_ERR_ARG; }
            ng = (uint32_t)g;
            nbk = ng * GRP_BPG;
            const uint64_t thr = fmh_threshold(c);
            unsigned __int128 mb = ((unsigned __int128)nbk << 64) / ((unsigned __int128)thr + 1);
            Mb = mb > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)mb;
            SYL_TRY(g_cnt.alloc(ng, st));
            SYL_CUDA(cudaMemsetAsync(g_cnt.p, 0, (size_t)ng * 4, st));
        }
        cap = expect_bases / c + expect_bases / (4 * c) + 65536;
        if (cap > expect_bases) cap = expect_bases + 16;
        // with groups cap is the overflow list, almost always empty: 1/16 of the estimate; a sample that
        // needs more (duplicate-heavy, homopolymers) is redone with the exact length
        if (ng) cap = cap / 16 + 65536;
        if (cap_override) cap = cap_override;
        if (ev_total() >= 0xFFFFFFFEull) { set_error("more than 2^32-2 survivor events in one sample"); return SYL_ERR_ARG; }
        SYL_TRY(b_ev.alloc(ev_total(), st));
        SYL_TRY(b_pend.alloc(ev_total(), st));
        SYL_CUDA(cudaMemsetAsync(ctx->d_counters, 0, 4 * sizeof(uint64_t), st));
        return SYL_OK;
    }

    // one batch of reads, device resident (ASCII bytes or 2-bit words); read indices continue from the
    // previous batch.  The seeding kernel appends the batch's events (hash, read, pair keys) to the event array.
    // rec_base: index of the batch's first read in the sample (batches may arrive in any order)
    int add(const uint8_t *d_bases, const uint32_t *d_packed, uint64_t nb, const uint64_t *d_off, uint64_t off_bias, uint64_t nr,
            uint64_t rec_base) {
        cudaStream_t st = ctx->stream;
        if (nr == 0) return SYL_OK;
        unsigned long long *dc = d_count();
        SYL_CUDA(cudaMemcpyAsync(dc + 3, dc + 1, 8, cudaMemcpyDeviceToDevice, st));  // pending entries before this batch
        SeedJob job;
        job.d_bases = d_bases; job.d_packed = d_packed; job.n_bases = nb; job.d_rec_off = d_off; job.off_bias = off_bias;
        job.n_rec = nr; job.k = k; job.c = c; job.sem = sem; job.with_pos = 0; job.d_out = b_ev.p; job.cap = cap;
        job.emit_events = 1; job.rec_base = rec_base; job.no_dedup = paired ? 2 : no_dedup; job.d_pend = b_pend.p;
        job.d_group_cnt = g_cnt.p; job.Mb = Mb; job.nbk = nbk; job.ng = ng; job.slot = slot; job.d_count = dc;
        SYL_TRY(seed_enqueue(ctx, job));
        if (!no_dedup && !paired && nb) {  // reads cut by a tile edge: their pair keys come from global memory
            const uint64_t n_words = (nb + 15) / 16;
            if (d_packed) k_events_fix<true><<<ctx->num_sms * 2, EV_THREADS, 0, st>>>(b_ev.p, b_pend.p, dc + 3, dc + 1, ev_total(), nullptr, d_packed, n_words, d_off, off_bias, rec_base);
            else k_events_fix<false><<<ctx->num_sms * 2, EV_THREADS, 0, st>>>(b_ev.p, b_pend.p, dc + 3, dc + 1, ev_total(), d_bases, nullptr, 0, d_off, off_bias, rec_base);
            ctx->launches++;
            SYL_CUDA(cudaGetLastError());
        }
        n_reads += nr;
        n_bases += nb;
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
        uint64_t *d_nruns = ctx->d_counters + 1;
        size_t rle_bytes = 0, scan_bytes = 0;
        cub::DeviceRunLengthEncode::Encode(nullptr, rle_bytes, hs, uniq.p, seg_len.p, d_nruns, N, st);
        cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, seg_len.p, seg_off.p, N, st);
        DevBuf<uint8_t> tmp2;
        SYL_TRY(tmp2.alloc(std::max(rle_bytes, scan_bytes), st));
        size_t tb = std::max(rle_bytes, scan_bytes);
        SYL_CUDA(cub::DeviceRunLengthEncode::Encode(tmp2.p, tb, hs, uniq.p, seg_len.p, d_nruns, N, st));
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + 1, d_nruns, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        const uint64_t U = ctx->h_counters[1];
        ctx->launches += 1;
        SYL_TRY(count.alloc(std::max<uint64_t>(U, 1), st));
        if (no_dedup && !paired) {
            k_copy_len<<<nblk(U, 256), 256, 0, st>>>(seg_len.p, count.p, U);
            ctx->launches++;
        } else {
            tb = std::max(rle_bytes, scan_bytes);
            SYL_CUDA(cub::DeviceScan::ExclusiveSum(tmp2.p, tb, seg_len.p, seg_off.p, U, st));
            DevBuf<uint64_t> set;
            SYL_TRY(set.alloc(2 * N, st));
            unsigned long long *d_ndup = reinterpret_cast<unsigned long long *>(ctx->d_counters + 2);
            SYL_CUDA(cudaMemsetAsync(d_ndup, 0, 8, st));
            if (paired) k_dedup_paired<<<nblk(U * 32, 128), 128, 0, st>>>(seg_off.p, seg_len.p, U, ord, ev_recflag, ev_p0, ev_p1, no_dedup, set.p, count.p, d_ndup);
            else k_dedup<<<nblk(U, 128), 128, 0, st>>>(seg_off.p, seg_len.p, U, ord, ev_recflag, ev_p0, ev_p1, set.p, count.p, d_ndup);
            ctx->launches += 2;
            SYL_CUDA(cudaGetLastError());
            SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + 2, d_ndup, 8, cudaMemcpyDeviceToHost, st));
            SYL_CUDA(cudaStreamSynchronize(st));
            *ndup_out = ctx->h_counters[2];
        }
        *U_out = U;
        return SYL_OK;
    }

    // need_cap: set when SYL_ERR_CAPACITY is returned (the true number of events)
    int finish(syl_sample **out, uint64_t *need_cap) {
        cudaStream_t st = ctx->stream;
        *need_cap = 0;
        syl_sample *s = new (std::nothrow) syl_sample();
        if (!s) return SYL_ERR_OOM;
        s->device = ctx->device;
        s->owner = ctx;
        s->stream = ctx->stream;
        s->k = k;
        s->c = c;
        s->mean_read_length = n_reads ? (double)n_bases / (double)n_reads : 0.;
        auto fail = [&](int rc) { syl_sample_free(s); return rc; };
#define SB_CUDA(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { set_error(std::string(#x) + ": " + cudaGetErrorString(_e)); return fail(_e == cudaErrorMemoryAllocation ? SYL_ERR_OOM : SYL_ERR_CUDA); } } while (0)
        if (n_reads == 0 || n_bases == 0) { *out = s; return SYL_OK; }
        unsigned long long *dc = d_count();
        EventRec *ev = b_ev.p;
        int rc;
        if (generic_postpass()) {
            SB_CUDA(cudaMemcpyAsync(ctx->h_counters, dc, 8, cudaMemcpyDeviceToHost, st));
            SB_CUDA(cudaStreamSynchronize(st));
            const uint64_t N = ctx->h_counters[0];
            if (N > cap) { *need_cap = N; syl_sample_free(s); return SYL_ERR_CAPACITY; }
            if (N == 0) { *out = s; return SYL_OK; }
            DevBuf<uint64_t> uq;
            DevBuf<uint32_t> ct;
            uint64_t U = 0, nd = 0;
            DevBuf<uint64_t> e_h, e_rf, e_p0, e_p1;
            if ((rc = e_h.alloc(N, st)) || (rc = e_rf.alloc(N, st)) || (rc = e_p0.alloc(N, st)) || (rc = e_p1.alloc(N, st))) return fail(rc);
            k_unpack_events<<<nblk(N, 256), 256, 0, st>>>(ev, N, e_h.p, e_rf.p, e_p0.p, e_p1.p);
            ctx->launches++;
            if ((rc = dedup_sorted(e_h.p, e_rf.p, e_p0.p, e_p1.p, N, uq, ct, &U, &nd)) != SYL_OK) return fail(rc);
            if ((rc = hblock_alloc(ctx, (void **)&s->hash, std::max<uint64_t>(U, 1) * 8))) return fail(rc);
            if ((rc = hblock_alloc(ctx, (void **)&s->count, std::max<uint64_t>(U, 1) * 4))) return fail(rc);
            SB_CUDA(cudaMemcpyAsync(s->hash, uq.p, U * 8, cudaMemcpyDeviceToDevice, st));
            SB_CUDA(cudaMemcpyAsync(s->count, ct.p, U * 4, cudaMemcpyDeviceToDevice, st));
            SB_CUDA(cudaStreamSynchronize(st));
            s->n = U;
            s->num_dup_removed = nd;
            *out = s;
            return SYL_OK;
        }
        // ---- primary path: CTA-local grouping / dedup of the group slots (ng, slot, Mb, g_cnt: begin()).
        // The kernels read the group counts from device memory.
        const uint64_t n_slots = (uint64_t)ng * slot;
        DevBuf<uint32_t> st_cnt, g_nuniq, g_n, uoff, fsz, foff, g_src, tmp_c;
        DevBuf<uint64_t> st_hash, tmp_h;
        DevBuf<uint8_t> g_fb;
        if ((rc = st_hash.alloc(n_slots, st)) || (rc = st_cnt.alloc(n_slots, st)) ||
            (rc = tmp_h.alloc(n_slots, st)) || (rc = tmp_c.alloc(n_slots, st)) ||  // in-kernel uniques: <= the slotted events
            (rc = g_nuniq.alloc(ng, st)) || (rc = g_n.alloc(ng, st)) ||
            (rc = g_fb.alloc(ng, st)) || (rc = uoff.alloc((uint64_t)ng + 1, st)) || (rc = fsz.alloc(ng, st)) ||
            (rc = foff.alloc((uint64_t)ng + 1, st)) || (rc = g_src.alloc(ng, st)))
            return fail(rc);
        unsigned long long *d_ndup = dc + 2;
        SB_CUDA(cudaFuncSetAttribute(k_group_dedup, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GroupSmem)));
        {
            KernelTimer kt(ctx, SYL_KERNEL_GROUP_DEDUP);
            k_group_dedup<<<ng, GRP_THREADS, sizeof(GroupSmem), st>>>(ev, g_cnt.p, slot, Mb, nbk, no_dedup,
                                                                       st_hash.p, st_cnt.p, g_nuniq.p, g_n.p, g_fb.p, d_ndup);
        }
        k_scan_u32<<<1, 1024, 0, st>>>(g_nuniq.p, ng, uoff.p);
        k_fallback_sizes<<<nblk(ng, 256), 256, 0, st>>>(g_n.p, g_fb.p, ng, fsz.p);
        k_scan_u32<<<1, 1024, 0, st>>>(fsz.p, ng, foff.p);
        k_compact_uniq<<<ng, 128, 0, st>>>(st_hash.p, st_cnt.p, slot, g_nuniq.p, uoff.p, g_fb.p, g_src.p, nullptr, nullptr,
                                            tmp_h.p, tmp_c.p);
        ctx->launches += 5;
        SB_CUDA(cudaGetLastError());
        SB_CUDA(cudaMemcpyAsync(ctx->h_counters, dc, 24, cudaMemcpyDeviceToHost, st));  // events, pending, duplicates
        SB_CUDA(cudaMemcpyAsync(ctx->h_counters + 4, uoff.p + ng, 4, cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaMemcpyAsync(ctx->h_counters + 5, foff.p + ng, 4, cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));  // the one synchronisation of a sketch
        const uint64_t N_ovf = ctx->h_counters[0];
        if (N_ovf > cap) { *need_cap = N_ovf; syl_sample_free(s); return SYL_ERR_CAPACITY; }
        // the overflow list holds only events of groups past their slot, all of which are fallback groups
        const uint64_t U1 = (uint32_t)ctx->h_counters[4], NF_slots = (uint32_t)ctx->h_counters[5], NF = NF_slots + N_ovf;
        uint64_t ndup = ctx->h_counters[2];
        static const bool dbg = getenv("SYL_DEBUG_TIMING") != nullptr;
        if (dbg) fprintf(stderr, "[sample post-pass] groups %u of %u slots, overflow list %llu (cap %llu): in-kernel uniques %llu, events handed to the generic path %llu (%.2f %% of the slotted events)\n",
                         ng, slot, (unsigned long long)N_ovf, (unsigned long long)cap, (unsigned long long)U1, (unsigned long long)NF,
                         n_slots ? 100.0 * (double)NF_slots / (double)n_slots : 0.);
        uint64_t U = U1;
        if (NF) {  // fallback groups through the generic path (heavy-hitter k-mers, duplicate-heavy replays)
            DevBuf<uint64_t> fh, f_rf, f_p0, f_p1, f_uq;
            DevBuf<uint32_t> f_ct;
            uint64_t U2 = 0, nd2 = 0;
            if ((rc = fh.alloc(NF, st)) || (rc = f_rf.alloc(NF, st)) || (rc = f_p0.alloc(NF, st)) || (rc = f_p1.alloc(NF, st)))
                return fail(rc);
            k_gather_fallback<<<ng, 256, 0, st>>>(ev, slot, g_n.p, g_fb.p, foff.p, fh.p, f_rf.p, f_p0.p, f_p1.p);
            ctx->launches++;
            if (N_ovf) {
                k_unpack_events<<<nblk(N_ovf, 256), 256, 0, st>>>(ev + n_slots, N_ovf, fh.p + NF_slots, f_rf.p + NF_slots,
                                                                  f_p0.p + NF_slots, f_p1.p + NF_slots);
                ctx->launches++;
            }
            if ((rc = dedup_sorted(fh.p, f_rf.p, f_p0.p, f_p1.p, NF, f_uq, f_ct, &U2, &nd2)) != SYL_OK) return fail(rc);
            ndup += nd2;
            U = U1 + U2;
            if ((rc = hblock_alloc(ctx, (void **)&s->hash, std::max<uint64_t>(U, 1) * 8))) return fail(rc);
            if ((rc = hblock_alloc(ctx, (void **)&s->count, std::max<uint64_t>(U, 1) * 4))) return fail(rc);
            if (U2) {  // slot the generic path's pairs into their groups' positions, compact straight into the result
                k_fallback_place<<<nblk(ng, 128), 128, 0, st>>>(g_fb.p, ng, nbk, Mb, f_uq.p, U2, g_nuniq.p, g_src.p);
                k_scan_u32<<<1, 1024, 0, st>>>(g_nuniq.p, ng, uoff.p);
                k_compact_uniq<<<ng, 128, 0, st>>>(st_hash.p, st_cnt.p, slot, g_nuniq.p, uoff.p, g_fb.p, g_src.p, f_uq.p, f_ct.p,
                                                    s->hash, s->count);
                ctx->launches += 3;
                SB_CUDA(cudaGetLastError());
            } else if (U) {
                SB_CUDA(cudaMemcpyAsync(s->hash, tmp_h.p, U * 8, cudaMemcpyDeviceToDevice, st));
                SB_CUDA(cudaMemcpyAsync(s->count, tmp_c.p, U * 4, cudaMemcpyDeviceToDevice, st));
            }
            SB_CUDA(cudaStreamSynchronize(st));  // f_uq / f_ct go out of scope
        } else {
            // exact-size result arrays; the copies are ordered on the ctx stream like every later use of the handle
            if ((rc = hblock_alloc(ctx, (void **)&s->hash, std::max<uint64_t>(U, 1) * 8))) return fail(rc);
            if ((rc = hblock_alloc(ctx, (void **)&s->count, std::max<uint64_t>(U, 1) * 4))) return fail(rc);
            if (U) {
                SB_CUDA(cudaMemcpyAsync(s->hash, tmp_h.p, U * 8, cudaMemcpyDeviceToDevice, st));
                SB_CUDA(cudaMemcpyAsync(s->count, tmp_c.p, U * 4, cudaMemcpyDeviceToDevice, st));
            }
        }
#undef SB_CUDA
        s->n = U;
        s->num_dup_removed = ndup;
        *out = s;
        return SYL_OK;
    }
};

}  // namespace syl

namespace syl {

// ---- host-memory ingest: pack on the host, ship 2-bit words ----------------------------------------
// ASCII bases in (pinned or pageable) host memory are cut into chunks on record boundaries; the ctx's
// worker pool packs chunk i+1.. into a ring of pinned staging buffers (exact BYTE_TO_SEQ codes, 16
// bases per word; record offsets rebased to u32) while chunk i crosses PCIe and earlier chunks are
// seeded.  4.3 bytes of H2D traffic per 16 bases instead of 16.5 (SURVEY §8 f3).  Chunks may also cross
// the link as ASCII, through a two-slot device ring: every chunk when packing is off (SYL_HOST_INGEST=ascii),
// else chunks taken from the back of the sample while the packers lag behind.
constexpr int ING_SLOTS = 4;
constexpr uint64_t ING_CHUNK = 32ull << 20;        // bases per packed chunk (multiple of 16)
constexpr uint64_t ING_ASCII_CHUNK = 128ull << 20; // bases per chunk when every chunk is shipped as ASCII
constexpr uint64_t ING_MAXREC = 1ull << 19;        // records per packed chunk
constexpr uint64_t ING_SLICE = 256ull << 10;       // bases per work item
constexpr uint64_t ING_OSLICE = 64ull << 10;       // offsets per work item
// SYL_INGEST_CHUNK overrides the chunk size of either mode (tests; read per call)
static uint64_t ingest_chunk(uint64_t dflt) {
    if (const char *e = getenv("SYL_INGEST_CHUNK")) {
        const long long v = atoll(e);
        if (v >= 16) return (uint64_t)v & ~15ull;
    }
    return dflt;
}

struct Chunk { uint64_t r0, r1, base, nb; };

// records [r0, r1) per chunk: at most max_bases bases and max_recs records, at least one record
static void plan_chunks(const uint64_t *rec_off, uint64_t n_reads, uint64_t max_bases, uint64_t max_recs,
                        std::vector<Chunk> &chunks) {
    uint64_t r0 = 0;
    while (r0 < n_reads) {
        const uint64_t base = rec_off[r0];
        uint64_t lo = r0 + 1, hi = std::min(n_reads, r0 + max_recs);
        while (lo < hi) {
            const uint64_t mid = (lo + hi + 1) >> 1;
            if (rec_off[mid] - base <= max_bases) lo = mid; else hi = mid - 1;
        }
        chunks.push_back({r0, lo, base, rec_off[lo] - base});
        r0 = lo;
    }
}

struct HostIngest {
    std::unique_ptr<PackPool> pool;
    cudaStream_t copy_stream = nullptr;  // the H2D copies of both rings
    // packed ring: words and chunk-relative u32 offsets, written by the pool
    uint32_t *h_words[ING_SLOTS] = {}, *h_off[ING_SLOTS] = {};  // pinned
    uint32_t *d_words[ING_SLOTS] = {}, *d_off32[ING_SLOTS] = {};
    uint64_t *d_off64[ING_SLOTS] = {};
    uint64_t cap_words = 0, cap_recs = 0;
    cudaEvent_t ev_copied[ING_SLOTS] = {}, ev_used[ING_SLOTS] = {};
    // ASCII ring: bases and u64 offsets copied from caller memory as they are
    uint8_t *d_asc[2] = {};
    uint64_t *d_aoff[2] = {};
    uint64_t cap_asc = 0, cap_aoff = 0;
    cudaEvent_t ev_a_copied[2] = {}, ev_a_used[2] = {};
    int a_slot = 0, a_last = -1;  // next ASCII slot; slot of the latest ASCII copy (-1: none yet)

    int init() {
        if (copy_stream) return SYL_OK;
        SYL_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
        for (int i = 0; i < ING_SLOTS; i++) {
            SYL_CUDA(cudaEventCreateWithFlags(&ev_copied[i], cudaEventDisableTiming));
            SYL_CUDA(cudaEventCreateWithFlags(&ev_used[i], cudaEventDisableTiming));
        }
        for (int i = 0; i < 2; i++) {
            SYL_CUDA(cudaEventCreateWithFlags(&ev_a_copied[i], cudaEventDisableTiming));
            SYL_CUDA(cudaEventCreateWithFlags(&ev_a_used[i], cudaEventDisableTiming));
        }
        return SYL_OK;
    }
    // the two streams that use the ring buffers: idle before a buffer is freed, and after a failed call
    void drain(cudaStream_t st) {
        cudaStreamSynchronize(st);
        cudaStreamSynchronize(copy_stream);
    }
    void free_packed() {
        for (int i = 0; i < ING_SLOTS; i++) {
            if (h_words[i]) cudaFreeHost(h_words[i]);
            if (h_off[i]) cudaFreeHost(h_off[i]);
            if (d_words[i]) cudaFree(d_words[i]);
            if (d_off32[i]) cudaFree(d_off32[i]);
            if (d_off64[i]) cudaFree(d_off64[i]);
            h_words[i] = h_off[i] = d_words[i] = d_off32[i] = nullptr;
            d_off64[i] = nullptr;
        }
        cap_words = cap_recs = 0;
    }
    void free_ascii() {
        for (int i = 0; i < 2; i++) {
            if (d_asc[i]) cudaFree(d_asc[i]);
            if (d_aoff[i]) cudaFree(d_aoff[i]);
            d_asc[i] = nullptr;
            d_aoff[i] = nullptr;
        }
        cap_asc = cap_aoff = 0;
    }
    // room for every chunk of the plan, and for at least ING_CHUNK bases and 65536 records
    int ensure_packed(cudaStream_t st, const std::vector<Chunk> &chunks) {
        uint64_t words = ING_CHUNK / 16, recs = 65536;
        for (const Chunk &c : chunks) {
            words = std::max(words, (c.nb + 15) / 16);
            recs = std::max(recs, c.r1 - c.r0 + 1);
        }
        if (words <= cap_words && recs <= cap_recs) return SYL_OK;
        drain(st);
        const uint64_t w = std::max(words, cap_words), r = std::max(recs, cap_recs);
        free_packed();
        for (int i = 0; i < ING_SLOTS; i++) {
            SYL_CUDA(cudaMallocHost((void **)&h_words[i], (w + 16) * 4));
            SYL_CUDA(cudaMallocHost((void **)&h_off[i], (r + 16) * 4));
            SYL_CUDA(cudaMalloc((void **)&d_words[i], (w + 16) * 4));
            SYL_CUDA(cudaMalloc((void **)&d_off32[i], (r + 16) * 4));
            SYL_CUDA(cudaMalloc((void **)&d_off64[i], (r + 16) * 8));
        }
        cap_words = w;
        cap_recs = r;
        return SYL_OK;
    }
    // room for every chunk of the plan, and for at least min_bases bases and 65536 records
    int ensure_ascii(cudaStream_t st, const std::vector<Chunk> &chunks, uint64_t min_bases) {
        uint64_t nb = min_bases, recs = 65536;
        for (const Chunk &c : chunks) {
            nb = std::max(nb, c.nb);
            recs = std::max(recs, c.r1 - c.r0 + 1);
        }
        if (nb <= cap_asc && recs <= cap_aoff) return SYL_OK;
        drain(st);
        nb = std::max(nb, cap_asc);
        recs = std::max(recs, cap_aoff);
        free_ascii();
        for (int i = 0; i < 2; i++) {
            SYL_CUDA(cudaMalloc((void **)&d_asc[i], nb + 256));  // the seeding kernel's bulk loads read past the last base
            SYL_CUDA(cudaMalloc((void **)&d_aoff[i], (recs + 16) * 8));
        }
        cap_asc = nb;
        cap_aoff = recs;
        return SYL_OK;
    }
    // One chunk from caller memory through the ASCII ring and into the builder.  The copy of a slot waits until
    // the previous chunk in it is seeded; the read indices travel with the chunk, so chunks may go in any order.
    int ship_ascii(syl_ctx *ctx, SampleBuilder &b, const uint8_t *bases, const uint64_t *rec_off, const Chunk &c) {
        const int slot = a_slot;
        a_slot ^= 1;
        const uint64_t nr = c.r1 - c.r0;
        cudaStreamWaitEvent(copy_stream, ev_a_used[slot], 0);
        if (cudaMemcpyAsync(d_asc[slot], bases + c.base, c.nb, cudaMemcpyHostToDevice, copy_stream) != cudaSuccess ||
            cudaMemcpyAsync(d_aoff[slot], rec_off + c.r0, (nr + 1) * 8, cudaMemcpyHostToDevice, copy_stream) != cudaSuccess) {
            set_error("H2D copy failed");
            return SYL_ERR_CUDA;
        }
        ctx->ingest_h2d_bytes += c.nb + (nr + 1) * 8;
        ctx->ingest_chunks_ascii++;
        cudaEventRecord(ev_a_copied[slot], copy_stream);
        cudaStreamWaitEvent(ctx->stream, ev_a_copied[slot], 0);
        const int rc = b.add(d_asc[slot], nullptr, c.nb, d_aoff[slot], c.base, nr, c.r0);
        cudaEventRecord(ev_a_used[slot], ctx->stream);
        a_last = slot;
        return rc;
    }
    ~HostIngest() {
        pool.reset();
        free_packed();
        free_ascii();
        for (int i = 0; i < ING_SLOTS; i++) {
            if (ev_copied[i]) cudaEventDestroy(ev_copied[i]);
            if (ev_used[i]) cudaEventDestroy(ev_used[i]);
        }
        for (int i = 0; i < 2; i++) {
            if (ev_a_copied[i]) cudaEventDestroy(ev_a_copied[i]);
            if (ev_a_used[i]) cudaEventDestroy(ev_a_used[i]);
        }
        if (copy_stream) cudaStreamDestroy(copy_stream);
    }
};

void ingest_destroy(syl_ctx *ctx) {
    delete static_cast<HostIngest *>(ctx->ingest);
    ctx->ingest = nullptr;
}

// host ASCII -> chunks -> builder.  ascii_only: every chunk crosses the link as it is, front to back (1 byte of
// H2D traffic per base, no host packing; pageable caller memory is fine).  Else the pool packs the chunks.
static int feed_host(syl_ctx *ctx, SampleBuilder &b, const uint8_t *bases, const uint64_t *rec_off, uint64_t n_reads,
                     bool ascii_only) {
    if (!ctx->ingest) ctx->ingest = new HostIngest();
    HostIngest &I = *static_cast<HostIngest *>(ctx->ingest);
    SYL_TRY(I.init());
    cudaStream_t st = ctx->stream, cs = I.copy_stream;
    std::vector<Chunk> chunks;
    if (ascii_only) {
        plan_chunks(rec_off, n_reads, ingest_chunk(ING_ASCII_CHUNK), n_reads, chunks);
        SYL_TRY(I.ensure_ascii(st, chunks, ING_ASCII_CHUNK));
        int rc = SYL_OK;
        for (size_t ci = 0; ci < chunks.size() && rc == SYL_OK; ci++) rc = I.ship_ascii(ctx, b, bases, rec_off, chunks[ci]);
        if (rc != SYL_OK) I.drain(st);
        return rc;
    }
    plan_chunks(rec_off, n_reads, ingest_chunk(ING_CHUNK), ING_MAXREC, chunks);
    for (const Chunk &c : chunks)  // the packed offsets are chunk-relative u32
        if (c.nb >= 0xFFFFFFF0ull) { set_error("a single record of 4 GB or more"); return SYL_ERR_ARG; }
    // Two resources work in parallel: the packers (host memory bandwidth / CPU quota) and the PCIe link.  Packed
    // chunks are consumed from the front in order; whenever the front chunk is not packed yet and no ASCII copy
    // is in flight, a chunk nobody has started is taken from the BACK and shipped as ASCII (4x the bytes, but the
    // link would idle otherwise).  Needs pinned caller memory (a pageable copy would block this thread).
    bool steal_ok = false;
    {
        cudaPointerAttributes pa;
        if (cudaPointerGetAttributes(&pa, bases) == cudaSuccess) steal_ok = pa.type == cudaMemoryTypeHost;
        else cudaGetLastError();
        const char *e = getenv("SYL_HOST_INGEST");
        if (e && std::string(e) == "packed-only") steal_ok = false;
    }
    SYL_TRY(I.ensure_packed(st, chunks));
    if (steal_ok) SYL_TRY(I.ensure_ascii(st, chunks, ING_CHUNK));
    if (!I.pool) I.pool.reset(new PackPool(default_pack_threads()));
    std::vector<PackItem> items;
    std::vector<uint32_t> chunk_items(chunks.size());
    for (size_t ci = 0; ci < chunks.size(); ci++) {
        const Chunk &c = chunks[ci];
        const int slot = (int)(ci % ING_SLOTS);
        uint32_t n_items = 0;
        for (uint64_t o = 0; o < c.nb; o += ING_SLICE, n_items++)
            items.push_back({bases + c.base + o, std::min(ING_SLICE, c.nb - o), I.h_words[slot] + o / 16, nullptr, 0, 0, nullptr, (uint32_t)ci});
        const uint64_t no = c.r1 - c.r0 + 1;
        for (uint64_t o = 0; o < no; o += ING_OSLICE, n_items++)
            items.push_back({nullptr, 0, nullptr, rec_off + c.r0 + o, c.base, std::min(ING_OSLICE, no - o), I.h_off[slot] + o, (uint32_t)ci});
        chunk_items[ci] = n_items;
    }
    I.pool->start(&items, &chunk_items, ING_SLOTS - 1);
    const bool force_steal = getenv("SYL_INGEST_FORCE_STEAL") != nullptr;  // tests: alternate packed / ASCII chunks
    int rc = SYL_OK;
    int64_t f = 0, bk = (int64_t)chunks.size() - 1, last_packed = -1;
    bool steal_turn = true;  // force_steal only: alternate ASCII and packed chunks
    while (f <= bk && rc == SYL_OK) {
        const bool steal_first = force_steal && steal_ok && steal_turn;
        if (!steal_first && I.pool->chunk_done((uint32_t)f)) {  // ---- packed chunk from the front
            const size_t ci = (size_t)f;
            const Chunk &c = chunks[ci];
            const int slot = (int)(ci % ING_SLOTS);
            const uint64_t nw = (c.nb + 15) / 16, no = c.r1 - c.r0 + 1;
            cudaStreamWaitEvent(cs, I.ev_used[slot], 0);  // the seeding of the previous chunk in this slot is done
            if (cudaMemcpyAsync(I.d_words[slot], I.h_words[slot], nw * 4, cudaMemcpyHostToDevice, cs) != cudaSuccess ||
                cudaMemcpyAsync(I.d_off32[slot], I.h_off[slot], no * 4, cudaMemcpyHostToDevice, cs) != cudaSuccess) {
                rc = SYL_ERR_CUDA; set_error("H2D copy failed"); break;
            }
            ctx->ingest_h2d_bytes += nw * 4 + no * 4;
            cudaEventRecord(I.ev_copied[slot], cs);
            cudaStreamWaitEvent(st, I.ev_copied[slot], 0);
            k_off32_to_64<<<nblk(no, 256), 256, 0, st>>>(I.d_off32[slot], no, I.d_off64[slot]);
            ctx->launches++;
            rc = b.add(nullptr, I.d_words[slot], c.nb, I.d_off64[slot], 0, c.r1 - c.r0, c.r0);
            cudaEventRecord(I.ev_used[slot], st);
            if (last_packed >= 0) {  // the pinned buffers of the previous packed chunk have crossed the link: refill them
                cudaEventSynchronize(I.ev_copied[last_packed % ING_SLOTS]);
                I.pool->open_gate(last_packed + ING_SLOTS);
            }
            last_packed = f;
            f++;
            ctx->ingest_chunks_packed++;
            steal_turn = true;
            continue;
        }
        const bool ascii_busy = !force_steal && I.a_last >= 0 && cudaEventQuery(I.ev_a_copied[I.a_last]) == cudaErrorNotReady;
        if (steal_ok && !ascii_busy && (!force_steal || steal_turn) && bk > f && I.pool->try_skip_chunk((uint32_t)bk)) {  // ---- ASCII chunk from the back
            rc = I.ship_ascii(ctx, b, bases, rec_off, chunks[(size_t)bk]);
            bk--;
            steal_turn = false;
            continue;
        }
        if (steal_first) { steal_turn = false; continue; }  // nothing to take from the back right now: go on with packed chunks
        // Front chunk still being packed.  If an ASCII copy is in flight and there are untouched chunks at the back,
        // whichever finishes first decides the next move (blocking on the packers alone would idle the link for as
        // long as they take: on a host whose memory system is shared by eight ranks that is most of the call).
        if (steal_ok && ascii_busy && bk > f) I.pool->wait_chunk_for((uint32_t)f, 40);
        else I.pool->wait_chunk((uint32_t)f);  // the packers are on it (or the only chunks left are theirs)
    }
    I.pool->open_gate((int64_t)1 << 60);  // all remaining items (skipped chunks included) drain
    I.pool->finish();
    static const bool dbg = getenv("SYL_DEBUG_TIMING") != nullptr;
    if (dbg) fprintf(stderr, "[host ingest] %zu chunks: %llu shipped as ASCII, %zu packed by %d threads\n", chunks.size(),
                     (unsigned long long)ctx->ingest_chunks_ascii, chunks.size() - (size_t)ctx->ingest_chunks_ascii, I.pool->threads());
    if (rc != SYL_OK) I.drain(st);
    return rc;
}

// packed: the input is 2-bit words (device or host memory); else ASCII
static int sketch_reads_impl(syl_ctx *ctx, int mem, const uint8_t *bases, const uint32_t *packed, uint64_t n_bases,
                             const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup, int sem, syl_sample **out) {
    if (!ctx || !out || (!bases && !packed && n_bases) || !rec_off) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (c == 0) { set_error("c must be >= 1"); return SYL_ERR_ARG; }
    if (mem != SYL_MEM_HOST && mem != SYL_MEM_DEVICE) { set_error("bad mem"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    // Host ASCII input: packed by the worker pool (fewer PCIe bytes) or shipped as it is.  Packing costs host memory
    // traffic (1.5 B per base: the packers read the ASCII, write the words, the copy engine reads them; ASCII costs 1 B
    // per base), so it pays while PCIe is the narrow resource — 1 to 4 processes per host — and loses once the ranks of
    // a host saturate its memory system instead (measured with 8 ranks on one host: 20.2 ms per 1 Gbp step shipping
    // ASCII, 32.7 ms packing; with 1 and 2 ranks packing wins, 10.2 vs 19.9 and 16.4 vs 19.9 ms).
    // SYL_HOST_INGEST = ascii | packed | packed-only overrides (read per call: the tests switch it at run time).
    const char *hi_env = getenv("SYL_HOST_INGEST");
    static const int local_ranks = []() { const char *e = getenv("LOCAL_WORLD_SIZE"); return e ? atoi(e) : 1; }();
    const bool host_ascii = hi_env ? std::string(hi_env) == "ascii" : local_ranks > 4;
    static const bool dbg = getenv("SYL_DEBUG_TIMING") != nullptr;
    auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    uint64_t cap_override = 0;
    for (int attempt = 0; attempt < 3; attempt++) {
        SampleBuilder b{ctx, k, c, no_dedup, sem};
        b.expect_bases = n_bases;
        b.expect_reads = n_reads;
        if (mem == SYL_MEM_HOST) ctx->ingest_h2d_bytes = ctx->ingest_chunks_packed = ctx->ingest_chunks_ascii = 0;
        SYL_TRY(b.begin(cap_override));
        const double t0 = now();
        int rc = SYL_OK;
        Staged<uint32_t> sp;   // host packed input staged whole
        Staged<uint64_t> so;
        if (mem == SYL_MEM_DEVICE) {
            rc = b.add(bases, packed, n_bases, rec_off, 0, n_reads, 0);
        } else if (packed) {
            const uint64_t nw = (n_bases + 15) / 16;
            SYL_TRY(sp.init(ctx, mem, packed, nw));
            SYL_TRY(so.init(ctx, mem, rec_off, n_reads + 1));
            ctx->ingest_h2d_bytes += nw * 4 + (n_reads + 1) * 8;
            rc = b.add(nullptr, sp.p, n_bases, so.p, 0, n_reads, 0);
        } else if (n_reads && n_bases) {
            rc = feed_host(ctx, b, bases, rec_off, n_reads, host_ascii);
        }
        if (rc != SYL_OK) return rc;
        const double t1 = now();
        uint64_t need = 0;
        rc = b.finish(out, &need);
        if (dbg) fprintf(stderr, "[syl_sketch_reads host] feed %.2f ms, finish %.2f ms (attempt %d)\n", t1 - t0, now() - t1, attempt);
        if (rc == SYL_ERR_CAPACITY) { cap_override = need + 16; continue; }  // more events than estimated: redo with the exact size
        return rc;
    }
    set_error("event capacity retry failed");
    return SYL_ERR_CAPACITY;
}

// One mate file of a paired sample: ASCII bytes or 2-bit words.
struct MateInput {
    const uint8_t *bases;
    const uint32_t *packed;
    uint64_t n_bases;
    const uint64_t *off;
    uint64_t n_words() const { return (n_bases + 15) / 16; }
};

// packed: both mates are 2-bit words (m1.packed / m2.packed), else ASCII (m1.bases / m2.bases)
static int sketch_read_pairs_impl(syl_ctx *ctx, int mem, bool packed, MateInput &m1, MateInput &m2, uint64_t n_pairs, int k,
                                  uint64_t c, int no_dedup, int sem, syl_sample **out) {
    if (!ctx || !out || (!m1.bases && !m1.packed && m1.n_bases) || (!m2.bases && !m2.packed && m2.n_bases) || !m1.off || !m2.off) {
        set_error("NULL argument");
        return SYL_ERR_ARG;
    }
    if (c == 0) { set_error("c must be >= 1"); return SYL_ERR_ARG; }
    if (mem != SYL_MEM_HOST && mem != SYL_MEM_DEVICE) { set_error("bad mem"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    Staged<uint8_t> sb[2];  // host memory: staged copies, alive until the call's sync
    Staged<uint32_t> sp[2];
    Staged<uint64_t> so[2];
    MateInput *m[2] = {&m1, &m2};
    for (int i = 0; i < 2; i++) {
        if (packed) { SYL_TRY(sp[i].init(ctx, mem, m[i]->packed, m[i]->n_words())); m[i]->packed = sp[i].p; }
        else { SYL_TRY(sb[i].init(ctx, mem, m[i]->bases, m[i]->n_bases)); m[i]->bases = sb[i].p; }
        SYL_TRY(so[i].init(ctx, mem, m[i]->off, n_pairs + 1));
        m[i]->off = so[i].p;
    }
    uint64_t cap_override = 0;
    for (int attempt = 0; attempt < 3; attempt++) {
        SampleBuilder b{ctx, k, c, no_dedup, sem};
        b.paired = true;
        b.expect_bases = m1.n_bases + m2.n_bases;
        b.expect_reads = 2 * n_pairs;
        SYL_TRY(b.begin(cap_override));
        unsigned long long *dc = b.d_count();
        // mate 1, then mate 2: both use the PAIR index as read index; the pending list tells the mates apart
        SYL_TRY(b.add(m1.bases, m1.packed, m1.n_bases, m1.off, 0, n_pairs, 0));
        SYL_CUDA(cudaMemcpyAsync(dc + 17, dc + 1, 8, cudaMemcpyDeviceToDevice, st));  // pending entries of mate 1
        SYL_TRY(b.add(m2.bases, m2.packed, m2.n_bases, m2.off, 0, n_pairs, 0));
        SYL_CUDA(cudaMemsetAsync(dc + 18, 0, 8, st));
        if (n_pairs) {
            auto fix = packed ? k_events_fix_paired<true> : k_events_fix_paired<false>;
            const uint64_t nw1 = packed ? m1.n_words() : 0, nw2 = packed ? m2.n_words() : 0;
            fix<<<ctx->num_sms * 2, EV_THREADS, 0, st>>>(b.b_ev.p, b.b_pend.p, dc + 18, dc + 17, b.cap, m1.bases, m1.packed, nw1,
                                                         m1.off, m2.bases, m2.packed, nw2, m2.off, 0, no_dedup);
            fix<<<ctx->num_sms * 2, EV_THREADS, 0, st>>>(b.b_ev.p, b.b_pend.p, dc + 17, dc + 1, b.cap, m1.bases, m1.packed, nw1,
                                                         m1.off, m2.bases, m2.packed, nw2, m2.off, 1, no_dedup);
            ctx->launches += 2;
            SYL_CUDA(cudaGetLastError());
        }
        b.n_reads = n_pairs;       // mean_read_length = mean length of mate 1 (src/sketch.rs:824-826)
        b.n_bases = m1.n_bases;
        uint64_t need = 0;
        const int rc = b.finish(out, &need);
        if (rc == SYL_ERR_CAPACITY) { cap_override = need + 16; continue; }
        if (rc == SYL_OK) SYL_CUDA(cudaStreamSynchronize(st));  // the staged inputs go out of scope
        return rc;
    }
    set_error("event capacity retry failed");
    return SYL_ERR_CAPACITY;
}

}  // namespace syl

using namespace syl;

extern "C" {

int syl_sketch_reads(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                     const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup,
                     int sem, syl_sample **out) {
    return sketch_reads_impl(ctx, mem, bases, nullptr, n_bases, rec_off, n_reads, k, c, no_dedup, sem, out);
}

int syl_sketch_reads_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                             const uint64_t *rec_off, uint64_t n_reads, int k, uint64_t c, int no_dedup,
                             int sem, syl_sample **out) {
    if (!packed && n_bases) { set_error("NULL argument"); return SYL_ERR_ARG; }
    return sketch_reads_impl(ctx, mem, nullptr, packed, n_bases, rec_off, n_reads, k, c, no_dedup, sem, out);
}

int syl_sketch_read_pairs(syl_ctx *ctx, int mem, const uint8_t *bases1, uint64_t n_bases1, const uint64_t *rec_off1,
                          const uint8_t *bases2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                          int k, uint64_t c, int no_dedup, int sem, syl_sample **out) {
    MateInput m1{bases1, nullptr, n_bases1, rec_off1}, m2{bases2, nullptr, n_bases2, rec_off2};
    return sketch_read_pairs_impl(ctx, mem, false, m1, m2, n_pairs, k, c, no_dedup, sem, out);
}

int syl_sketch_read_pairs_packed2(syl_ctx *ctx, int mem, const uint32_t *packed1, uint64_t n_bases1, const uint64_t *rec_off1,
                                  const uint32_t *packed2, uint64_t n_bases2, const uint64_t *rec_off2, uint64_t n_pairs,
                                  int k, uint64_t c, int no_dedup, int sem, syl_sample **out) {
    MateInput m1{nullptr, packed1, n_bases1, rec_off1}, m2{nullptr, packed2, n_bases2, rec_off2};
    return sketch_read_pairs_impl(ctx, mem, true, m1, m2, n_pairs, k, c, no_dedup, sem, out);
}

int syl_pack_threads(void) { return default_pack_threads(); }

int syl_ctx_ingest_stats(const syl_ctx *ctx, uint64_t *h2d_bytes, uint64_t *chunks_packed, uint64_t *chunks_ascii) {
    if (!ctx) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (h2d_bytes) *h2d_bytes = ctx->ingest_h2d_bytes;
    if (chunks_packed) *chunks_packed = ctx->ingest_chunks_packed;
    if (chunks_ascii) *chunks_ascii = ctx->ingest_chunks_ascii;
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
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    syl_sample *s = new (std::nothrow) syl_sample();
    if (!s) return SYL_ERR_OOM;
    s->device = ctx->device; s->owner = ctx; s->stream = st; s->k = k; s->c = c; s->n = n;
    auto fill = [&]() -> int {  // any failure below frees the handle and its blocks
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
        return SYL_OK;
    };
    const int frc = fill();
    if (frc != SYL_OK) { syl_sample_free(s); return frc; }
    *out = s;
    return SYL_OK;
}

uint64_t syl_sample_size(const syl_sample *s) { return s ? s->n : 0; }
double syl_sample_mean_read_length(const syl_sample *s) { return s ? s->mean_read_length : 0.; }
uint64_t syl_sample_num_dup_removed(const syl_sample *s) { return s ? s->num_dup_removed : 0; }
void syl_sample_set_mean_read_length(syl_sample *s, double v) { if (s) s->mean_read_length = v; }

int syl_sample_download(syl_ctx *ctx, const syl_sample *s, uint64_t *hash, uint32_t *count) {
    if (!ctx || !s) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
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
