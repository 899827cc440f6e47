// seed_kernel.cuh — the seeding kernel template (see seed.cu for the formulation).
#pragma once
#include "common.cuh"

namespace syl {

constexpr int SEED_THREADS = 256;
#ifndef SEED_TILE_CFG
#define SEED_TILE_CFG 32768
#endif
#ifndef SEED_MINB_CFG
#define SEED_MINB_CFG 4
#endif
constexpr int SEED_TILE = SEED_TILE_CFG;   // window-start positions (== bases) per CTA
constexpr int SEED_W_MAX = 32;     // most windows per thread-run (candidate bit mask is 32 bits)
constexpr int SEED_W_MIN = 24;     // run lengths W instantiated: 24, 30, 32 (template parameter)
constexpr int SEED_HALO = 48;      // bytes staged past the tile (>= k-1, multiple of 16)
constexpr int SEED_STAGE = SEED_TILE >= 32768 ? 512 : 256;    // survivors staged per CTA before falling back to global atomics
constexpr int SEED_CAND = SEED_TILE >= 32768 ? 1024 : 512;    // candidate windows buffered per record chunk (overflow is handled inline)
constexpr int SEED_RUNS_PER_THREAD = (SEED_TILE / SEED_W_MIN + 2 * SEED_THREADS - 1) / SEED_THREADS;
constexpr int SEED_MAXRUNS = SEED_THREADS * SEED_RUNS_PER_THREAD;  // >= SEED_TILE / SEED_W_MIN + SEED_THREADS
static_assert(SEED_MAXRUNS >= SEED_TILE / SEED_W_MIN + SEED_THREADS, "run table too small");
constexpr int SEED_ASC_BYTES = SEED_TILE + SEED_HALO;  // 32816, multiple of 16
constexpr int SEED_NCHUNK16 = SEED_ASC_BYTES / 16;     // 2051 16-base words per stream
constexpr int SEED_FW_WORDS = SEED_NCHUNK16 + 1 + 8;   // +1 leading pad word, +8 slack for run loads
constexpr int SEED_CW_WORDS = SEED_NCHUNK16 + 8;
constexpr int SEED_PK_WORDS = (SEED_NCHUNK16 + 3) & ~3;  // 2-bit input: words staged per tile (whole 16-byte groups)
static_assert(SEED_TILE % 64 == 0, "2-bit tiles must start on 16-byte boundaries");

struct SeedSmem {
    // region A: staging of the ASCII bytes (or, for 2-bit input, of the packed words); after packing
    // it is reused for the per-chunk record table and the survivor staging buffer (see offsets below)
    alignas(128) uint8_t asc[SEED_ASC_BYTES + 16];
    alignas(16) uint32_t fw[SEED_FW_WORDS];
    alignas(16) uint32_t cw[SEED_CW_WORDS];
    alignas(16) uint8_t lut[4][256];  // lut[j][b] = BYTE_TO_SEQ[b] << (6 - 2j)
    alignas(8) unsigned long long mbar;
};
// views into region A once the ASCII bytes are dead
struct SeedMeta {
    long long rel[SEED_THREADS];      // rec_off[r] - tile_start (may be very negative)
    int s0[SEED_THREADS];             // first valid window start inside the tile (tile-relative)
    int cnt[SEED_THREADS];            // number of valid window starts inside the tile
    int len[SEED_THREADS];            // record length (saturated), for the pair-key rule
    int rbase[SEED_THREADS + 1];      // exclusive scan of ceil(cnt / W)
    int warp_tot[SEED_THREADS / 32];
    unsigned int stage_count;
    unsigned int cand_count;
    unsigned long long flush_base;
    alignas(16) EventRec stage[SEED_STAGE];  // holds syl_survivor (16 B) or EventRec (32 B) entries
    uint32_t cand[SEED_CAND];          // (tile-relative window start << 8) | record slot
    uint16_t run_rec[SEED_MAXRUNS];    // run -> record slot + 1 (filled by a max-scan over run starts)
};
static_assert(sizeof(SeedMeta) <= SEED_ASC_BYTES, "meta must fit in the dead ASCII region");
static_assert(SEED_TILE <= 65536, "tile-relative window starts are kept as u16");
// survivors (16 B) fill only the lower half of the 32-byte staging entries; the upper half keeps each
// staged survivor's tile-relative window start
__device__ __forceinline__ uint16_t *seed_stage_pos(SeedMeta &M) {
    return reinterpret_cast<uint16_t *>(reinterpret_cast<syl_survivor *>(M.stage) + SEED_STAGE);
}

// Where an emitted event goes (read-sketch post-pass, sample.cu).  Group g of the post-pass owns the
// GRP_BPG consecutive hash buckets [g * GRP_BPG, (g + 1) * GRP_BPG), bucket = min(mulhi(hash, Mb), nbk - 1),
// and the fixed slot out[g * slot, (g + 1) * slot): the flush writes every event straight into its group.
// An event past its slot's capacity is appended to the overflow list out[ng * slot ..) at the running
// counter *g_count; its group then takes the post-pass's generic path.  cnt == nullptr: no groups, every
// event is appended at *g_count (read pairs, SYL_SAMPLE_POSTPASS=sort).  Appends past cap are counted
// but dropped; the caller compares the final count with cap and redoes the sample.
struct GroupOut {
    uint32_t *cnt;  // events per group (can exceed slot)
    uint64_t Mb;
    uint32_t nbk, ng, slot;
    // position of the event in out, or ~0ull when it is dropped
    __device__ __forceinline__ uint64_t place(uint64_t h, unsigned long long *g_count, uint64_t cap) const {
        if (cnt) {
            uint32_t g = (uint32_t)__umul64hi(h, Mb);
            g = (g < nbk ? g : nbk - 1) / GRP_BPG;
            const uint32_t i = atomicAdd(&cnt[g], 1u);
            if (i < slot) return (uint64_t)g * slot + i;
        }
        const unsigned long long gi = atomicAdd(g_count, 1ull);
        return gi < cap ? (uint64_t)ng * slot + gi : ~0ull;  // ng * slot == 0 without groups
    }
};

// The constants 1 and 0, passed as kernel parameters so that ptxas cannot fold the hot loop's
// predicated IMADs (x * one + zero) back into ALU-pipe moves.  The padding keeps k_seed's parameter
// offsets where its register allocation was tuned: ptxas allocates differently without it, and the
// W = 24 kernels then spill 8-12 bytes.
struct ImadConst { uint32_t pad_[3], one, zero; };

// Slotted survivor output (genome sketching): tile t writes its survivors to out[t * cap ..) and their
// number to tile_cnt[t] instead of appending at a global counter, so that the output is already in tile
// (= position) order and no global sort is needed.  cap == 0: off.  A tile with more survivors than the
// slot (or the CTA's staging buffer) holds raises *overflow; the caller then takes the generic path.
struct SlotOut { uint32_t cap; uint32_t *tile_cnt; uint32_t *overflow; };

// 64-bit multiply by a 32-bit constant as IMAD.WIDE + IMAD (2 FMA-pipe instructions)
__device__ __forceinline__ void mul64c(uint32_t lo, uint32_t hi, uint32_t c, uint32_t &plo, uint32_t &phi) {
    uint64_t t;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(t) : "r"(lo), "r"(c));
    plo = (uint32_t)t;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(phi) : "r"(hi), "r"(c), "r"((uint32_t)(t >> 32)));
}

// x ^= x >> s on halves: 2 SHF + 2 LOP3 (ALU pipe)
template <int SH>
__device__ __forceinline__ void xorshift(uint32_t &lo, uint32_t &hi, uint32_t extra_hi) {
    const uint32_t sh = hi >> SH, sl = __funnelshift_r(lo, hi, SH);
    lo ^= sl;
    hi = hi ^ sh ^ extra_hi;
}

// High 32 bits of mm_hash64 (src/seeding.rs:4-15) on a k-mer given as two 32-bit halves.
//   * the NOT of step 1 is folded into the first xor-shift: for X = ~x,
//       (X ^ X>>24).lo = x.lo ^ (x>>24).lo            (the complements cancel)
//       (X ^ X>>24).hi = x.hi ^ (x.hi>>24) ^ 0xFFFFFF00
//   * only the high word of the last multiply is formed; survivors re-derive the full hash
__device__ __forceinline__ uint32_t hash_hi32(uint32_t lo, uint32_t hi) {
    uint32_t a, b;
    mul64c(lo, hi, 0x200001u, a, b);
    xorshift<24>(a, b, 0xFFFFFF00u);
    mul64c(a, b, 265u, lo, hi);
    xorshift<14>(lo, hi, 0u);
    mul64c(lo, hi, 21u, a, b);
    xorshift<28>(a, b, 0u);
    return __umulhi(a, 0x80000001u) + b * 0x80000001u;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// 32 consecutive bases (64 bits, MSB-first) of the forward stream starting at tile-relative base q
__device__ __forceinline__ uint64_t fw64(const SeedSmem &S, uint32_t q) {
    const uint32_t bitpos = 32u + 2u * q, w = bitpos >> 5, sh = bitpos & 31u;
    const uint32_t a = S.fw[w], b = S.fw[w + 1], c = S.fw[w + 2];
    return ((uint64_t)__funnelshift_l(b, a, sh) << 32) | __funnelshift_l(c, b, sh);
}

// The hot loop: one run of W windows starting at tile-relative window start p of the streams fw / cw.
// Returns the candidate mask (bit i: the high word of window p+i's hash is <= thr_hi).  Only the high
// word of the hash is formed; candidates (1/c of windows) are collected in a bit mask, so the loop
// has no divergent code.
template <int K, int W>
__device__ __forceinline__ uint32_t seed_run(const uint32_t *fw, const uint32_t *cw, int p, uint32_t thr_hi, const ImadConst ic) {
    constexpr uint32_t PAD = 64 - 2 * K;                     // unused high bits of a k-mer word
    constexpr uint32_t HI_MASK = (1u << (32 - PAD)) - 1u;    // K=31: 0x3FFFFFFF, K=21: 0x3FF
    // realign the two streams so that window i of this run starts at bit 2i
    uint32_t F[4], G[4];
    {
        const uint32_t bitpos = 32u + 2u * (uint32_t)p - PAD;
        const uint32_t q0 = bitpos >> 5, sh = bitpos & 31u;
        uint32_t w0 = fw[q0], w1 = fw[q0 + 1], w2 = fw[q0 + 2], w3 = fw[q0 + 3], w4 = fw[q0 + 4];
        F[0] = __funnelshift_l(w1, w0, sh);
        F[1] = __funnelshift_l(w2, w1, sh);
        F[2] = __funnelshift_l(w3, w2, sh);
        F[3] = __funnelshift_l(w4, w3, sh);
        const uint32_t cq = (uint32_t)p >> 4, csh = ((uint32_t)p & 15u) * 2u;
        uint32_t c0 = cw[cq], c1 = cw[cq + 1], c2 = cw[cq + 2], c3 = cw[cq + 3], c4 = cw[cq + 4];
        G[0] = __funnelshift_r(c0, c1, csh);
        G[1] = __funnelshift_r(c1, c2, csh);
        G[2] = __funnelshift_r(c2, c3, csh);
        G[3] = __funnelshift_r(c3, c4, csh);
    }
    uint32_t cand = 0u;
#pragma unroll
    for (int i = 0; i < W; i++) {
        const int jb = (2 * i) >> 5;
        const uint32_t sft = (uint32_t)((2 * i) & 31);
        const uint32_t f_hi = __funnelshift_l(F[jb + 1], F[jb], sft) & HI_MASK;
        const uint32_t f_lo = __funnelshift_l(F[jb + 2], F[jb + 1], sft);
        const uint32_t r_lo = __funnelshift_r(G[jb], G[jb + 1], sft);
        const uint32_t r_hi = __funnelshift_r(G[jb + 1], G[jb + 2], sft) & HI_MASK;
        // canonical k-mer = min(forward, reverse complement), src/seeding.rs:131-136.  Both are
        // < 2^62, so as IEEE doubles they are finite, non-negative and ordered like the
        // integers: ONE compare on the FP64 pipe replaces the two-instruction 64-bit integer
        // compare on the ALU pipe, which is this loop's limiter.  The select is a pair of
        // predicated IMADs (FMA pipe).
        uint32_t c_lo = r_lo, c_hi = r_hi;
        asm("{\n\t.reg .pred p;\n\t.reg .f64 a, b;\n\tmov.b64 a, {%2, %3};\n\tmov.b64 b, {%4, %5};\n\t"
            "setp.lt.f64 p, a, b;\n\t@p mad.lo.u32 %0, %2, %6, %7;\n\t@p mad.lo.u32 %1, %3, %6, %7;\n\t}"
            : "+r"(c_lo), "+r"(c_hi) : "r"(f_lo), "r"(f_hi), "r"(r_lo), "r"(r_hi), "r"(ic.one), "r"(ic.zero));
        const uint32_t hh = hash_hi32(c_lo, c_hi);
        // candidate bit set by a predicated IMAD (FMA pipe): the bits are distinct, so add == or
        asm("{\n\t.reg .pred p;\n\tsetp.le.u32 p, %1, %2;\n\t@p mad.lo.u32 %0, %3, %4, %0;\n\t}"
            : "+r"(cand) : "r"(hh), "r"(thr_hi), "r"(ic.one), "r"(1u << i));
    }
    return cand;
}

// Exact re-derivation of one candidate window: k-mer halves from the packed streams at an arbitrary
// position, full 64-bit hash, threshold test, survivor staged in shared memory.
// EMIT == 0: 16-byte syl_survivor (hash, record, position).
// EMIT == 1: 32-byte EventRec for the read-sketch post-pass, including pair_kmer_single's keys
//            (src/sketch.rs:624-656) taken straight from the packed stream when the read's first 32
//            bases and the 32 bases from its middle are inside the staged tile (99 % of 150 bp
//            reads); otherwise the event is flagged EV_PENDING and k_events_fix fills the keys.
template <int K, int EMIT>
__device__ __forceinline__ void seed_resolve(const SeedSmem &S, SeedMeta &M, uint32_t pw, int j, uint64_t rc, uint64_t thr,
                                             void *__restrict__ out, uint64_t cap,
                                             unsigned long long *__restrict__ g_count, uint64_t rec_base, int no_dedup,
                                             uint32_t *__restrict__ pend, const GroupOut go) {
    constexpr uint32_t PAD = 64 - 2 * K;
    constexpr uint32_t HI_MASK = (1u << (32 - PAD)) - 1u;
    const uint32_t bitpos = 32u + 2u * pw - PAD;
    const uint32_t q0 = bitpos >> 5, sh = bitpos & 31u;
    const uint32_t w0 = S.fw[q0], w1 = S.fw[q0 + 1], w2 = S.fw[q0 + 2];
    const uint64_t f = ((uint64_t)(__funnelshift_l(w1, w0, sh) & HI_MASK) << 32) | __funnelshift_l(w2, w1, sh);
    const uint32_t cq = pw >> 4, csh = (pw & 15u) * 2u;
    const uint32_t c0 = S.cw[cq], c1 = S.cw[cq + 1], c2 = S.cw[cq + 2];
    const uint64_t rr = ((uint64_t)(__funnelshift_r(c1, c2, csh) & HI_MASK) << 32) | __funnelshift_r(c0, c1, csh);
    const uint64_t h = mm_hash64(f < rr ? f : rr);  // src/seeding.rs:131-137
    if (h >= thr) return;                           // src/seeding.rs:139
    const unsigned int idx = atomicAdd(&M.stage_count, 1u);
    if (EMIT == 0) {
        syl_survivor sv;
        sv.hash = h;
        sv.rec = (uint32_t)(rc + (uint64_t)j);
        sv.pos = (uint32_t)((long long)pw - M.rel[j] + (K - 1));
        if (idx < (unsigned)SEED_STAGE) {
            reinterpret_cast<syl_survivor *>(M.stage)[idx] = sv;
            seed_stage_pos(M)[idx] = (uint16_t)pw;  // tile-relative window start: the slotted flush ranks by it
        } else {
            const unsigned long long gi = atomicAdd(g_count, 1ull);
            if (gi < cap) reinterpret_cast<syl_survivor *>(out)[gi] = sv;
        }
    } else {
        EventRec ev;
        ev.hash = h;
        const int L = M.len[j];
        const bool has_pair = !no_dedup && L <= 400 && L >= 66;  // src/sketch.rs:923, :627
        // no_dedup == 2: read pairs — the keys need both mates, every event is completed by k_events_fix_paired
        ev.recflag = ((rec_base + rc + (uint64_t)j) << 1) | (no_dedup == 2 ? EV_PENDING : (has_pair ? 0ull : NO_PAIR));
        ev.p0 = 0;
        ev.p1 = 0;
        if (has_pair) {
            const long long st = M.rel[j];  // read start, tile-relative
            const long long mid = st + (L >> 1);
            if (st >= 0 && mid + 32 <= (long long)SEED_NCHUNK16 * 16) {
                const uint64_t a = fw64(S, (uint32_t)st), b = fw64(S, (uint32_t)mid);
                const uint32_t kf = even_fields(a), kg = even_fields(a << 2);  // s[0,2,..,30] / s[1,3,..,31]
                const uint32_t kr = even_fields(b), kt = even_fields(b << 2);
                ev.p0 = ((uint64_t)kf << 32) | kr;  // doublepairs.0 = [kmer_f, kmer_r]
                ev.p1 = ((uint64_t)kg << 32) | kt;  // doublepairs.1 = [kmer_g, kmer_t]
            } else {
                ev.recflag |= EV_PENDING;
            }
        }
        if (idx < (unsigned)SEED_STAGE) {
            M.stage[idx] = ev;
        } else {
            const uint64_t pos = go.place(ev.hash, g_count, cap);
            if (pos != ~0ull) {
                reinterpret_cast<EventRec *>(out)[pos] = ev;
                if (ev.recflag & EV_PENDING) pend[atomicAdd(g_count + 1, 1ull)] = (uint32_t)pos;
            }
        }
    }
}

// PACKED: the input is 2-bit codes (16 bases per little-endian u32, base 16w+j in bits [30-2j, 31-2j],
// i.e. exactly the forward stream), made by the host packer (host_pack.cpp) from the reference's
// BYTE_TO_SEQ table.  The staging copies a quarter of the bytes and the pack phase shrinks to the
// complement stream; everything after it is the same as for ASCII input.
template <int K, int EMIT, int W, bool PACKED>
__global__ void __launch_bounds__(SEED_THREADS, SEED_MINB_CFG)
k_seed(const uint8_t *__restrict__ bases, uint64_t n_bases, const uint64_t *__restrict__ rec_off, uint64_t off_bias,
       const uint32_t *__restrict__ tile_rec, uint64_t thr, int sem, int with_pos,
       void *__restrict__ out, uint64_t cap, unsigned long long *__restrict__ g_count,
       const ImadConst ic, uint64_t rec_base, int no_dedup, uint32_t *__restrict__ pend, const GroupOut go, const SlotOut slot) {
    static_assert(W >= SEED_W_MIN && W <= SEED_W_MAX, "run length");
    extern __shared__ __align__(128) uint8_t smem_raw[];
    SeedSmem &S = *reinterpret_cast<SeedSmem *>(smem_raw);
    SeedMeta &M = *reinterpret_cast<SeedMeta *>(S.asc);

    const int tid = threadIdx.x;
    const uint64_t T0 = (uint64_t)blockIdx.x * SEED_TILE;
    const uint64_t T1 = T0 + SEED_TILE;
    const uint32_t thr_hi = (uint32_t)(thr >> 32);

    // ---- stage the tile: TMA bulk copy for the 16-byte-aligned body, plain loads for the tail.
    //      ASCII: SEED_ASC_BYTES bytes from bases + T0; PACKED: SEED_PK_WORDS words from word T0 / 16.
    constexpr uint32_t UNIT = PACKED ? 4u : 1u;                    // bytes per staged element
    constexpr uint32_t NSTAGE = PACKED ? SEED_PK_WORDS : SEED_ASC_BYTES;
    const uint64_t e0 = PACKED ? T0 / 16 : T0;
    const uint64_t remain = (PACKED ? (n_bases + 15) / 16 : n_bases) - e0;
    const uint32_t avail = remain < (uint64_t)NSTAGE ? (uint32_t)remain : NSTAGE;
    const uint32_t nbulk = avail & ~(16u / UNIT - 1u);             // elements in whole 16-byte groups
    const uint32_t mbar = smem_u32(&S.mbar);
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0 && nbulk) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(nbulk * UNIT)
                     : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(S.asc)),
            "l"(bases + e0 * UNIT), "r"(nbulk * UNIT), "r"(mbar)
            : "memory");
    }
    // tail (< 16 bytes) and zero fill of everything past the end of the buffer
    if (PACKED) {
        const uint32_t *words = reinterpret_cast<const uint32_t *>(bases);
        for (uint32_t i = nbulk + tid; i < NSTAGE; i += SEED_THREADS)
            reinterpret_cast<uint32_t *>(S.asc)[i] = (i < avail) ? words[e0 + i] : 0u;
    } else {
        for (uint32_t i = nbulk + tid; i < (uint32_t)SEED_ASC_BYTES + 16; i += SEED_THREADS)
            S.asc[i] = (i < avail) ? bases[T0 + i] : (uint8_t)0;
        const uint32_t code = byte_to_seq((uint32_t)tid);
        S.lut[0][tid] = (uint8_t)(code << 6);
        S.lut[1][tid] = (uint8_t)(code << 4);
        S.lut[2][tid] = (uint8_t)(code << 2);
        S.lut[3][tid] = (uint8_t)code;
    }
    if (tid < 8) {
        S.fw[SEED_NCHUNK16 + 1 + tid] = 0u;
        S.cw[SEED_NCHUNK16 + tid] = 0u;
    }
    if (tid == 0) S.fw[0] = 0u;
    if (nbulk) {
        uint32_t done = 0;
        while (!done) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(mbar)
                : "memory");
        }
    }
    __syncthreads();

    // ---- pack: 16 bases -> one forward word (MSB-first) + one complement word (LSB-first).
    // ASCII, per byte: one PRMT (extract) + one LDS.U8 from the pre-shifted table; per 4 bytes two 3-input
    // ORs.  PACKED: the staged word is the forward word.
    for (int ch = tid; ch < SEED_NCHUNK16; ch += SEED_THREADS) {
        uint32_t f;
        if (PACKED) {
            f = reinterpret_cast<const uint32_t *>(S.asc)[ch];
        } else {
            const uint4 v = *reinterpret_cast<const uint4 *>(S.asc + 16 * ch);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
            uint32_t g[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const uint32_t b0 = __byte_perm(w[q], 0u, 0x4440), b1 = __byte_perm(w[q], 0u, 0x4441);
                const uint32_t b2 = __byte_perm(w[q], 0u, 0x4442), b3 = __byte_perm(w[q], 0u, 0x4443);
                g[q] = ((uint32_t)S.lut[0][b0] | (uint32_t)S.lut[1][b1] | (uint32_t)S.lut[2][b2]) | (uint32_t)S.lut[3][b3];
            }
            const uint32_t lo16 = __byte_perm(g[3], g[2], 0x0040), hi16 = __byte_perm(g[1], g[0], 0x0040);
            f = __byte_perm(lo16, hi16, 0x5410);
        }
        // complement stream: base j's (3 - code) at bits [2j, 2j+2): reverse the 16 fields of f
        uint32_t x = __brev(f);                                        // fields reversed, bits swapped in each
        x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);       // swap bits back inside each field
        S.fw[1 + ch] = f;
        S.cw[ch] = ~x;
    }
    __syncthreads();  // the staged input is dead from here on; region A becomes SeedMeta

    if (tid == 0) M.stage_count = 0u;

    const uint32_t r_lo = tile_rec[blockIdx.x];
    const uint32_t r_hi = tile_rec[blockIdx.x + 1];  // inclusive
    const int lane = tid & 31, wid = tid >> 5;

    for (uint64_t rc = r_lo; rc <= (uint64_t)r_hi; rc += SEED_THREADS) {
        // -- per-record table for this chunk of (up to) SEED_THREADS records
        int runs = 0;
        const uint64_t r = rc + tid;
        if (r <= (uint64_t)r_hi) {
            const uint64_t a = rec_off[r] - off_bias, b = rec_off[r + 1] - off_bias;
            const uint64_t L = b - a;
            const uint64_t nv = valid_windows(L, (uint32_t)K, sem, with_pos);
            const uint64_t lo = a > T0 ? a : T0;
            uint64_t hi = a + nv;
            if (hi > T1) hi = T1;
            const int cnt = hi > lo ? (int)(hi - lo) : 0;
            M.rel[tid] = (long long)a - (long long)T0;
            M.s0[tid] = (int)(lo - T0);
            M.cnt[tid] = cnt;
            M.len[tid] = L > 0x7FFFFFFFull ? 0x7FFFFFFF : (int)L;
            runs = (cnt + W - 1) / W;
        }
        // block-wide exclusive scan of runs
        int incl = runs;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) M.warp_tot[wid] = incl;
        __syncthreads();
        int wbase = 0;
#pragma unroll
        for (int w = 0; w < SEED_THREADS / 32; w++) wbase += (w < wid) ? M.warp_tot[w] : 0;
        M.rbase[tid] = wbase + incl - runs;
        if (tid == SEED_THREADS - 1) M.rbase[SEED_THREADS] = wbase + incl;
        __syncthreads();
        const int total = M.rbase[SEED_THREADS];

        // -- run -> record table: every record with runs marks its first run with (slot + 1); an
        //    inclusive max-scan then spreads the marker over the record's runs (markers increase
        //    with the run index), so a thread finds its record with one byte load instead of a
        //    binary search per run.
        {
            const int base5 = tid * SEED_RUNS_PER_THREAD;
#pragma unroll
            for (int e = 0; e < SEED_RUNS_PER_THREAD; e++) M.run_rec[base5 + e] = 0;
            __syncthreads();
            if (runs > 0) M.run_rec[M.rbase[tid]] = (uint16_t)(tid + 1);
            __syncthreads();
            int v[SEED_RUNS_PER_THREAD], m = 0;
#pragma unroll
            for (int e = 0; e < SEED_RUNS_PER_THREAD; e++) { m = max(m, (int)M.run_rec[base5 + e]); v[e] = m; }
            int inc = m;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) inc = max(inc, __shfl_up_sync(0xffffffffu, inc, d));
            int excl = __shfl_up_sync(0xffffffffu, inc, 1);
            if (lane == 0) excl = 0;
            if (lane == 31) M.warp_tot[wid] = inc;
            __syncthreads();
            int wmax = 0;
#pragma unroll
            for (int w = 0; w < SEED_THREADS / 32; w++) wmax = max(wmax, (w < wid) ? M.warp_tot[w] : 0);
            const int pre = max(excl, wmax);
#pragma unroll
            for (int e = 0; e < SEED_RUNS_PER_THREAD; e++) M.run_rec[base5 + e] = (uint16_t)max(v[e], pre);
            if (tid == 0) M.cand_count = 0u;
            __syncthreads();
        }

        // -- one run of <= W windows per thread per pass
        for (int q = tid; q < total; q += SEED_THREADS) {
            const int j = (int)M.run_rec[q] - 1;
            const int ridx = q - M.rbase[j];
            const int p = M.s0[j] + ridx * W;            // tile-relative first window start
            const int n = min(W, M.cnt[j] - ridx * W);
            uint32_t cand = seed_run<K, W>(S.fw, S.cw, p, thr_hi, ic);
            if (n < W) cand &= (1u << n) - 1u;  // n >= 1 (windows past n belong to the next run / record)
            // candidates go to a CTA-wide list and are re-derived exactly by all threads afterwards
            while (cand) {
                const int i = __ffs(cand) - 1;
                cand &= cand - 1u;
                const unsigned int ci = atomicAdd(&M.cand_count, 1u);
                if (ci < (unsigned)SEED_CAND) {
                    M.cand[ci] = ((uint32_t)(p + i) << 8) | (uint32_t)j;
                } else {  // list full (tiny c): resolve inline
                    seed_resolve<K, EMIT>(S, M, (uint32_t)(p + i), j, rc, thr, out, cap, g_count, rec_base, no_dedup, pend, go);
                }
            }
        }
        __syncthreads();
        {
            const unsigned int nc = min(M.cand_count, (unsigned)SEED_CAND);
            for (unsigned int ci = tid; ci < nc; ci += SEED_THREADS) {
                const uint32_t e = M.cand[ci];
                seed_resolve<K, EMIT>(S, M, e >> 8, (int)(e & 255u), rc, thr, out, cap, g_count, rec_base, no_dedup, pend, go);
            }
        }
        __syncthreads();  // table is rewritten by the next chunk
    }

    // ---- flush staged survivors: one global atomic per CTA, coalesced 16-byte stores
    __syncthreads();
    if (EMIT == 0 && slot.cap) {  // slotted output: this tile's slot, no atomics (launcher passes cap = 0, so nothing was appended)
        const unsigned int total = M.stage_count;
        const unsigned int lim = min((unsigned)SEED_STAGE, slot.cap);
        const unsigned int nst = min(total, lim);
        if (tid == 0) {
            slot.tile_cnt[blockIdx.x] = nst;
            if (total > lim) atomicExch(slot.overflow, 1u);
        }
        // The slot is written in POSITION order (the genome post-pass then needs no sort at all): bitmap of the
        // staged window starts in the dead stream words, rank = survivors before the word + bits below.
        constexpr int NW = SEED_TILE / 32, PER = NW / SEED_THREADS;
        static_assert(NW % SEED_THREADS == 0 && NW <= SEED_CW_WORDS, "bitmap layout");
        uint32_t *bits = S.fw, *pre = S.cw;
        const uint16_t *sp = seed_stage_pos(M);
        for (int i = tid; i < NW; i += SEED_THREADS) bits[i] = 0u;
        __syncthreads();
        for (unsigned int i = tid; i < nst; i += SEED_THREADS) atomicOr(&bits[sp[i] >> 5], 1u << (sp[i] & 31u));
        __syncthreads();
        {
            uint32_t cnt[PER], tot = 0;
#pragma unroll
            for (int e = 0; e < PER; e++) { cnt[e] = __popc(bits[PER * tid + e]); tot += cnt[e]; }
            uint32_t inc = tot;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d); if ((tid & 31) >= d) inc += v; }
            if ((tid & 31) == 31) M.warp_tot[tid >> 5] = (int)inc;
            __syncthreads();
            uint32_t base = inc - tot;
            for (int w = 0; w < (tid >> 5); w++) base += (uint32_t)M.warp_tot[w];
#pragma unroll
            for (int e = 0; e < PER; e++) { pre[PER * tid + e] = base; base += cnt[e]; }
        }
        __syncthreads();
        syl_survivor *dst = reinterpret_cast<syl_survivor *>(out) + (uint64_t)blockIdx.x * slot.cap;
        for (unsigned int i = tid; i < nst; i += SEED_THREADS) {
            const uint32_t p = sp[i], w = p >> 5;
            dst[pre[w] + __popc(bits[w] & ((1u << (p & 31u)) - 1u))] = reinterpret_cast<const syl_survivor *>(M.stage)[i];
        }
        return;
    }
    const unsigned int staged = min(M.stage_count, (unsigned)SEED_STAGE);
    if (EMIT == 1 && go.cnt) {  // events straight into their post-pass groups
        for (unsigned int i = tid; i < staged; i += SEED_THREADS) {
            const EventRec ev = M.stage[i];
            const uint64_t pos = go.place(ev.hash, g_count, cap);
            if (pos == ~0ull) continue;
            reinterpret_cast<EventRec *>(out)[pos] = ev;
            // reads cut by the tile edge: pair keys are filled in by k_events_fix
            if (ev.recflag & EV_PENDING) pend[atomicAdd(g_count + 1, 1ull)] = (uint32_t)pos;
        }
        return;
    }
    if (tid == 0 && staged) M.flush_base = atomicAdd(g_count, (unsigned long long)staged);
    __syncthreads();
    if (staged) {
        const unsigned long long base = M.flush_base;
        for (unsigned int i = tid; i < staged; i += SEED_THREADS) {
            if (base + i >= cap) continue;
            if (EMIT == 0) reinterpret_cast<syl_survivor *>(out)[base + i] = reinterpret_cast<const syl_survivor *>(M.stage)[i];
            else {
                const EventRec ev = M.stage[i];
                reinterpret_cast<EventRec *>(out)[base + i] = ev;
                // reads cut by the tile edge: pair keys are filled in by k_events_fix
                if (ev.recflag & EV_PENDING) pend[atomicAdd(g_count + 1, 1ull)] = (uint32_t)(base + i);
            }
        }
    }
}


using seed_kern_t = void (*)(const uint8_t *, uint64_t, const uint64_t *, uint64_t, const uint32_t *, uint64_t, int, int,
                             void *, uint64_t, unsigned long long *, const ImadConst, uint64_t, int, uint32_t *, const GroupOut, const SlotOut);

// One translation unit per (K, EMIT) instantiates the three run lengths for ASCII and 2-bit input and
// exports a getter, so the 24 kernels compile in parallel.
#define SEED_DEFINE_KERNELS(NAME, K, EMIT)                                              \
    seed_kern_t NAME(int W, bool packed) {                                              \
        switch (W) {                                                                    \
            case 24: return packed ? k_seed<K, EMIT, 24, true> : k_seed<K, EMIT, 24, false>; \
            case 30: return packed ? k_seed<K, EMIT, 30, true> : k_seed<K, EMIT, 30, false>; \
            default: return packed ? k_seed<K, EMIT, 32, true> : k_seed<K, EMIT, 32, false>; \
        }                                                                               \
    }

seed_kern_t seed_kernels_k31_sv(int W, bool packed);
seed_kern_t seed_kernels_k31_ev(int W, bool packed);
seed_kern_t seed_kernels_k21_sv(int W, bool packed);
seed_kern_t seed_kernels_k21_ev(int W, bool packed);

}  // namespace syl
