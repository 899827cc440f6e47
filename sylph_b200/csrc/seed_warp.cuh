// seed_warp.cuh — the seeding kernel, warp-autonomous persistent formulation (k_seed_w).
//
// Same arithmetic as k_seed (seed_kernel.cuh: 2-bit streams, record-aware runs, FP64-pipe canonical
// compare, hash on the FMA + ALU pipes, candidates re-derived exactly), different control structure:
//   * the grid is persistent (CTAs/SM x SMs); every WARP is an independent worker that claims
//     tiles of SW_TW window starts from a global counter and owns a private shared-memory slab
//     (TMA destination, the two packed streams, record / run tables, candidate and survivor
//     staging).  After start-up there is no __syncthreads: a warp never waits for another warp, so
//     the stage / pack / table / resolve / flush phases of one warp overlap the hot loops of the
//     others at warp granularity instead of CTA granularity (k_seed: ALU pipe 73 % busy with 1.6
//     warps per issue slot parked at CTA barriers).
//   * the TMA bulk copy of the NEXT tile is issued as soon as the current tile is packed (the ASCII
//     buffer is dead from then on), so its latency hides behind the hot loop.
//   * PACKED input: the tile arrives as 2-bit codes (16 bases per little-endian u32, base 16w+j in
//     bits [30-2j, 31-2j], i.e. exactly the forward stream), produced by the host packer
//     (host_pack.cu) from the reference's BYTE_TO_SEQ table; the pack phase shrinks to a copy plus
//     the complement stream.  H2D traffic drops 4x.
#pragma once
#include "seed_kernel.cuh"

namespace syl {

#ifndef SEEDW_TW
#define SEEDW_TW 3584
#endif
#ifndef SEEDW_MINB
#define SEEDW_MINB 3
#endif
#ifndef SEEDW_WARPS
#define SEEDW_WARPS 8
#endif
constexpr int SW_TW = SEEDW_TW;                 // capacity: most window starts (== bases) per warp-tile; the launcher picks
                                                // the actual tile length tw <= SW_TW so that a tile holds just under 32 r runs
constexpr int SW_HALO = 48;                     // bases staged past the tile (>= k-1, multiple of 16)
constexpr int SW_WARPS = SEEDW_WARPS;
constexpr int SW_THREADS = 32 * SW_WARPS;
constexpr int SW_ASC = SW_TW + SW_HALO;         // bytes / bases staged per tile (multiple of 16)
constexpr int SW_NCH = SW_ASC / 16;             // 16-base words per stream
constexpr int SW_NCHP = (SW_NCH + 3) & ~3;      // packed input: words copied per tile (16-byte multiple)
constexpr int SW_STAGE = SW_TW / 128;           // survivors staged per tile (expected: TW/250); overflow -> global appends
constexpr int SW_CAND = 2 * SW_STAGE;           // candidate windows buffered per record chunk; overflow -> inline
constexpr int SW_RPL = (SW_TW / SEED_W_MIN + 32 + 31) / 32;  // run-table entries per lane
constexpr int SW_MAXRUNS = 32 * SW_RPL;         // >= TW / W_MIN + 32 (every record adds at most one partial run)
static_assert(SW_TW % 16 == 0 && SW_STAGE >= 8, "tile size");

template <bool PACKED>
struct alignas(128) SeedWSlab {
    alignas(128) uint8_t asc[PACKED ? SW_NCHP * 4 : SW_ASC + 16];  // TMA destination: ASCII bytes, or 2-bit words for packed input
    alignas(16) uint32_t fwbuf[4 + SW_NCHP + 8];           // [3] = lead pad word, [4..] = forward stream
    alignas(16) uint32_t cw[SW_NCHP + 8];                  // complement stream, LSB-first
    alignas(16) EventRec stage[SW_STAGE];                  // syl_survivor (16 B) or EventRec (32 B) entries
    long long rel[32];                                     // rec_off[r] - tile start (may be very negative)
    int s0[32], cnt[32], len[32], rbase[33];               // per record of the current chunk (see k_seed)
    uint32_t cand[SW_CAND];                                // (tile-relative window start << 8) | record slot
    uint8_t run_rec[SW_MAXRUNS];                           // run -> record slot + 1
    unsigned int stage_count, cand_count;
    alignas(8) unsigned long long mbar;
};

struct SeedWArgs {
    const uint8_t *bases;      // ASCII input (PACKED == false)
    const uint32_t *packed;    // 2-bit input (PACKED == true), ceil(n_bases / 16) words
    uint64_t n_bases;
    const uint64_t *rec_off;
    uint64_t off_bias;
    const uint32_t *tile_rec;  // first record overlapping each tile (n_tiles + 1 entries)
    uint64_t n_tiles;
    uint32_t tw;               // window starts per tile (multiple of 64, <= SW_TW)
    uint64_t thr;
    int sem, with_pos;
    void *out;                 // syl_survivor[cap] or EventRec[cap]
    uint64_t cap;
    unsigned long long *g_count;  // running number of survivors / events in `out` (not reset per launch by the kernel)
    unsigned long long *g_pend;   // running number of entries in `pend`
    unsigned long long *g_tile;   // tile claim counter, zero at launch
    ShiftMul smul;
    uint64_t rec_base;
    int no_dedup;
    uint32_t *pend;
    GroupOut go;               // events: post-pass groups (see seed_kernel.cuh)
};

// one run of W windows starting at tile-relative window start p: candidate bit mask (bit i: high word of
// the hash of window p+i is <= the high word of the threshold).  Same instruction mix as k_seed's loop.
template <int K, int VAR, int W>
__device__ __forceinline__ uint32_t seedw_run(const uint32_t *fw, const uint32_t *cwp, int p,
                                              uint32_t thr_hi, const ShiftMul smul) {
    constexpr uint32_t PAD = 64 - 2 * K;
    constexpr uint32_t HI_MASK = (1u << (32 - PAD)) - 1u;
    uint32_t F[4], G[4];
    {
        const uint32_t bitpos = 32u + 2u * (uint32_t)p - PAD;
        const uint32_t q0 = bitpos >> 5, sh = bitpos & 31u;
        const uint32_t w0 = fw[q0], w1 = fw[q0 + 1], w2 = fw[q0 + 2], w3 = fw[q0 + 3], w4 = fw[q0 + 4];
        F[0] = __funnelshift_l(w1, w0, sh);
        F[1] = __funnelshift_l(w2, w1, sh);
        F[2] = __funnelshift_l(w3, w2, sh);
        F[3] = __funnelshift_l(w4, w3, sh);
        const uint32_t cq = (uint32_t)p >> 4, csh = ((uint32_t)p & 15u) * 2u;
        const uint32_t c0 = cwp[cq], c1 = cwp[cq + 1], c2 = cwp[cq + 2], c3 = cwp[cq + 3], c4 = cwp[cq + 4];
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
        // canonical k-mer (src/seeding.rs:131-136): both values < 2^62, so ONE FP64 compare orders them;
        // select and candidate bit as predicated IMADs (FMA pipe) — see seed_kernel.cuh
        uint32_t c_lo = r_lo, c_hi = r_hi;
        asm("{\n\t.reg .pred p;\n\t.reg .f64 a, b;\n\tmov.b64 a, {%2, %3};\n\tmov.b64 b, {%4, %5};\n\t"
            "setp.lt.f64 p, a, b;\n\t@p mad.lo.u32 %0, %2, %6, %7;\n\t@p mad.lo.u32 %1, %3, %6, %7;\n\t}"
            : "+r"(c_lo), "+r"(c_hi) : "r"(f_lo), "r"(f_hi), "r"(r_lo), "r"(r_hi), "r"(smul.one), "r"(smul.zero));
        const uint32_t hh = hash_hi32<VAR>(c_lo, c_hi, smul);
        asm("{\n\t.reg .pred p;\n\tsetp.le.u32 p, %1, %2;\n\t@p mad.lo.u32 %0, %3, %4, %0;\n\t}"
            : "+r"(cand) : "r"(hh), "r"(thr_hi), "r"(smul.one), "r"(1u << i));
    }
    return cand;
}

// 32 consecutive bases (64 bits, MSB-first) of a forward stream starting at tile-relative base q
__device__ __forceinline__ uint64_t seedw_fw64(const uint32_t *fw, uint32_t q) {
    const uint32_t bitpos = 32u + 2u * q, w = bitpos >> 5, sh = bitpos & 31u;
    const uint32_t a = fw[w], b = fw[w + 1], c = fw[w + 2];
    return ((uint64_t)__funnelshift_l(b, a, sh) << 32) | __funnelshift_l(c, b, sh);
}

// exact re-derivation of one candidate window (see seed_resolve in seed_kernel.cuh), warp-slab version
template <int K, int EMIT, bool PACKED>
__device__ __forceinline__ void seedw_resolve(SeedWSlab<PACKED> &S, const SeedWArgs &A, uint32_t pw, int j, uint64_t rc) {
    constexpr uint32_t PAD = 64 - 2 * K;
    constexpr uint32_t HI_MASK = (1u << (32 - PAD)) - 1u;
    const uint32_t *fw = S.fwbuf + 3;
    const uint32_t bitpos = 32u + 2u * pw - PAD;
    const uint32_t q0 = bitpos >> 5, sh = bitpos & 31u;
    const uint32_t w0 = fw[q0], w1 = fw[q0 + 1], w2 = fw[q0 + 2];
    const uint64_t f = ((uint64_t)(__funnelshift_l(w1, w0, sh) & HI_MASK) << 32) | __funnelshift_l(w2, w1, sh);
    const uint32_t cq = pw >> 4, csh = (pw & 15u) * 2u;
    const uint32_t c0 = S.cw[cq], c1 = S.cw[cq + 1], c2 = S.cw[cq + 2];
    const uint64_t rr = ((uint64_t)(__funnelshift_r(c1, c2, csh) & HI_MASK) << 32) | __funnelshift_r(c0, c1, csh);
    const uint64_t h = mm_hash64(f < rr ? f : rr);  // src/seeding.rs:131-137
    if (h >= A.thr) return;                         // src/seeding.rs:139
    const unsigned int idx = atomicAdd(&S.stage_count, 1u);
    if (EMIT == 0) {
        syl_survivor sv;
        sv.hash = h;
        sv.rec = (uint32_t)(rc + (uint64_t)j);
        sv.pos = (uint32_t)((long long)pw - S.rel[j] + (K - 1));
        if (idx < (unsigned)SW_STAGE) {
            reinterpret_cast<syl_survivor *>(S.stage)[idx] = sv;
        } else {
            const unsigned long long gi = atomicAdd(A.g_count, 1ull);
            if (gi < A.cap) reinterpret_cast<syl_survivor *>(A.out)[gi] = sv;
        }
    } else {
        EventRec ev;
        ev.hash = h;
        const int L = S.len[j];
        const bool has_pair = !A.no_dedup && L <= 400 && L >= 66;  // src/sketch.rs:923, :627
        // no_dedup == 2: read pairs — the keys need both mates, every event is completed by k_events_fix_paired
        ev.recflag = ((A.rec_base + rc + (uint64_t)j) << 1) | (A.no_dedup == 2 ? EV_PENDING : (has_pair ? 0ull : NO_PAIR));
        ev.p0 = 0;
        ev.p1 = 0;
        if (has_pair) {
            const long long st = S.rel[j];  // read start, tile-relative
            const long long mid = st + (L >> 1);
            if (st >= 0 && mid + 32 <= (long long)A.tw + SW_HALO) {
                const uint64_t a = seedw_fw64(fw, (uint32_t)st), b = seedw_fw64(fw, (uint32_t)mid);
                const uint32_t kf = even_fields(a), kg = even_fields(a << 2);  // s[0,2,..,30] / s[1,3,..,31]
                const uint32_t kr = even_fields(b), kt = even_fields(b << 2);
                ev.p0 = ((uint64_t)kf << 32) | kr;  // doublepairs.0 = [kmer_f, kmer_r]
                ev.p1 = ((uint64_t)kg << 32) | kt;  // doublepairs.1 = [kmer_g, kmer_t]
            } else {
                ev.recflag |= EV_PENDING;
            }
        }
        if (idx < (unsigned)SW_STAGE) {
            S.stage[idx] = ev;
        } else {
            const uint64_t pos = A.go.place(ev.hash, A.g_count, A.cap);
            if (pos != ~0ull) {
                reinterpret_cast<EventRec *>(A.out)[pos] = ev;
                if (ev.recflag & EV_PENDING) A.pend[atomicAdd(A.g_pend, 1ull)] = (uint32_t)pos;
            }
        }
    }
}

template <int K, int VAR, int EMIT, int W, bool PACKED>
__global__ void __launch_bounds__(SW_THREADS, SEEDW_MINB)
k_seed_w(const SeedWArgs A) {
    static_assert(W >= SEED_W_MIN && W <= SEED_W_MAX, "run length");
    extern __shared__ __align__(128) uint8_t smem_raw[];
    uint8_t(*lut)[256] = reinterpret_cast<uint8_t(*)[256]>(smem_raw);  // lut[j][b] = BYTE_TO_SEQ[b] << (6 - 2j)
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    SeedWSlab<PACKED> &S = *reinterpret_cast<SeedWSlab<PACKED> *>(smem_raw + 1024 + (size_t)wid * sizeof(SeedWSlab<PACKED>));
    uint32_t *const fw = S.fwbuf + 3;  // fw[0] = lead pad word, fw[1 + ch] = bases 16ch .. 16ch+15 (MSB-first)
    const uint32_t thr_hi = (uint32_t)(A.thr >> 32);
    const uint32_t mbar = smem_u32(&S.mbar);
    const uint32_t asc_n = A.tw + SW_HALO;          // bases staged per tile
    const int nch = (int)(asc_n >> 4);              // 16-base words per stream
    const uint32_t nchp = ((uint32_t)nch + 3u) & ~3u;  // packed input: words copied per tile (16-byte multiple)

    if (!PACKED) {
        for (int b = tid; b < 256; b += SW_THREADS) {
            const uint32_t code = byte_to_seq((uint32_t)b);
            lut[0][b] = (uint8_t)(code << 6);
            lut[1][b] = (uint8_t)(code << 4);
            lut[2][b] = (uint8_t)(code << 2);
            lut[3][b] = (uint8_t)code;
        }
    }
    if (lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fw[0] = 0u;
    }
    for (int i = nch + lane; i < SW_NCHP + 8; i += 32) {  // words past the staged bases: read by run loads, never used
        fw[1 + i] = 0u;
        S.cw[i] = 0u;
    }
    __syncthreads();  // the only CTA-wide barrier: lut and mbarriers are ready

    // stage tile t into this warp's slab: one TMA bulk copy for the 16-byte-aligned body (lane 0),
    // plain loads for the tail of the buffer's last tile
    auto issue_load = [&](uint64_t t) {
        const uint64_t T0 = t * (uint64_t)A.tw;
        if (!PACKED) {
            const uint64_t remain = A.n_bases - T0;
            const uint32_t avail = remain < (uint64_t)asc_n ? (uint32_t)remain : asc_n;
            const uint32_t nbulk = avail & ~15u;
            if (avail < asc_n)
                for (uint32_t i = nbulk + lane; i < asc_n + 16; i += 32) S.asc[i] = (i < avail) ? A.bases[T0 + i] : (uint8_t)0;
            __syncwarp();
            if (lane == 0) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(nbulk) : "memory");
                if (nbulk)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                     smem_u32(S.asc)), "l"(A.bases + T0), "r"(nbulk), "r"(mbar) : "memory");
            }
        } else {
            const uint64_t w0 = T0 >> 4, n_words = (A.n_bases + 15) >> 4;
            const uint64_t remain = n_words - w0;
            const uint32_t avail = remain < (uint64_t)nchp ? (uint32_t)remain : nchp;
            const uint32_t nbulk = avail & ~3u;  // whole 16-byte groups
            if (avail < nchp)
                for (uint32_t i = nbulk + lane; i < nchp; i += 32)
                    reinterpret_cast<uint32_t *>(S.asc)[i] = (i < avail) ? A.packed[w0 + i] : 0u;
            __syncwarp();
            if (lane == 0) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(nbulk * 4u) : "memory");
                if (nbulk)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                     smem_u32(S.asc)), "l"(A.packed + w0), "r"(nbulk * 4u), "r"(mbar) : "memory");
            }
        }
    };
    uint32_t phase = 0;
    uint64_t t;
    {
        unsigned long long t_l0 = 0;
        if (lane == 0) t_l0 = atomicAdd(A.g_tile, 1ull);
        t = __shfl_sync(0xffffffffu, t_l0, 0);
    }
    if (t < A.n_tiles) issue_load(t);
    while (t < A.n_tiles) {
        // claim the next tile now; the atomic's result is only needed after the pack phase
        unsigned long long tn_l0 = 0;
        if (lane == 0) tn_l0 = atomicAdd(A.g_tile, 1ull);
        const uint64_t T0 = t * (uint64_t)A.tw, T1 = T0 + A.tw;
        {   // wait for the bulk copy of tile t
            uint32_t done = 0;
            while (!done) {
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(done) : "r"(mbar), "r"(phase) : "memory");
            }
            phase ^= 1u;
        }
        if (!PACKED) {
            // pack: 16 ASCII bytes -> one forward word (MSB-first) + one complement word (LSB-first); see k_seed
            for (int ch = lane; ch < nch; ch += 32) {
                const uint4 v = *reinterpret_cast<const uint4 *>(S.asc + 16 * ch);
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
                uint32_t g[4];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const uint32_t b0 = __byte_perm(w[q], 0u, 0x4440), b1 = __byte_perm(w[q], 0u, 0x4441);
                    const uint32_t b2 = __byte_perm(w[q], 0u, 0x4442), b3 = __byte_perm(w[q], 0u, 0x4443);
                    g[q] = ((uint32_t)lut[0][b0] | (uint32_t)lut[1][b1] | (uint32_t)lut[2][b2]) | (uint32_t)lut[3][b3];
                }
                const uint32_t lo16 = __byte_perm(g[3], g[2], 0x0040), hi16 = __byte_perm(g[1], g[0], 0x0040);
                const uint32_t f = __byte_perm(lo16, hi16, 0x5410);
                uint32_t x = __brev(f);
                x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
                fw[1 + ch] = f;
                S.cw[ch] = ~x;
            }
        } else {
            // forward stream = the staged words; complement stream: reverse the 16 fields of a word, complement
            for (int ch = lane; ch < (int)nchp; ch += 32) {
                const uint32_t f = reinterpret_cast<const uint32_t *>(S.asc)[ch];
                uint32_t x = __brev(f);
                x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
                fw[1 + ch] = f;
                S.cw[ch] = ~x;
            }
        }
        __syncwarp();  // the staging buffer is dead: the next tile may land while this one is processed
        const uint64_t tn = __shfl_sync(0xffffffffu, tn_l0, 0);
        if (tn < A.n_tiles) issue_load(tn);
        if (lane == 0) S.stage_count = 0u;

        const uint32_t r_lo = A.tile_rec[t];
        const uint32_t r_hi = A.tile_rec[t + 1];  // inclusive
        for (uint64_t rc = r_lo; rc <= (uint64_t)r_hi; rc += 32) {
            // -- record table for this chunk of (up to) 32 records: one record per lane
            int runs = 0;
            const uint64_t r = rc + lane;
            if (r <= (uint64_t)r_hi) {
                const uint64_t a = A.rec_off[r] - A.off_bias, b = A.rec_off[r + 1] - A.off_bias;
                const uint64_t L = b - a;
                const uint64_t nv = valid_windows(L, (uint32_t)K, A.sem, A.with_pos);
                const uint64_t lo = a > T0 ? a : T0;
                uint64_t hi = a + nv;
                if (hi > T1) hi = T1;
                const int cnt = hi > lo ? (int)(hi - lo) : 0;
                S.rel[lane] = (long long)a - (long long)T0;
                S.s0[lane] = (int)(lo - T0);
                S.cnt[lane] = cnt;
                S.len[lane] = L > 0x7FFFFFFFull ? 0x7FFFFFFF : (int)L;
                runs = (cnt + W - 1) / W;
            }
            int incl = runs;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += v;
            }
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            S.rbase[lane] = incl - runs;
            if (lane == 0) S.cand_count = 0u;
            // run -> record table: first run of every record is marked with (slot + 1); an inclusive
            // max-scan spreads the marker over the record's runs
            const int base_e = lane * SW_RPL;
#pragma unroll
            for (int e = 0; e < SW_RPL; e++) S.run_rec[base_e + e] = 0;
            __syncwarp();
            if (runs > 0) S.run_rec[incl - runs] = (uint8_t)(lane + 1);
            __syncwarp();
            {
                int v[SW_RPL], m = 0;
#pragma unroll
                for (int e = 0; e < SW_RPL; e++) { m = max(m, (int)S.run_rec[base_e + e]); v[e] = m; }
                int inc = m;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) inc = max(inc, __shfl_up_sync(0xffffffffu, inc, d));
                int pre = __shfl_up_sync(0xffffffffu, inc, 1);
                if (lane == 0) pre = 0;
#pragma unroll
                for (int e = 0; e < SW_RPL; e++) S.run_rec[base_e + e] = (uint8_t)max(v[e], pre);
            }
            __syncwarp();

            // -- one run of <= W windows per lane per pass
            for (int q = lane; q < total; q += 32) {
                const int j = (int)S.run_rec[q] - 1;
                const int ridx = q - S.rbase[j];
                const int p = S.s0[j] + ridx * W;  // tile-relative first window start
                const int n = min(W, S.cnt[j] - ridx * W);
                uint32_t cand = seedw_run<K, VAR, W>(fw, S.cw, p, thr_hi, A.smul);
                if (n < W) cand &= (1u << n) - 1u;  // n >= 1
                while (cand) {
                    const int i = __ffs(cand) - 1;
                    cand &= cand - 1u;
                    const unsigned int ci = atomicAdd(&S.cand_count, 1u);
                    if (ci < (unsigned)SW_CAND) S.cand[ci] = ((uint32_t)(p + i) << 8) | (uint32_t)j;
                    else seedw_resolve<K, EMIT, PACKED>(S, A, (uint32_t)(p + i), j, rc);  // list full (tiny c): inline
                }
            }
            __syncwarp();
            {
                const unsigned int nc = min(S.cand_count, (unsigned)SW_CAND);
                for (unsigned int ci = lane; ci < nc; ci += 32) {
                    const uint32_t e = S.cand[ci];
                    seedw_resolve<K, EMIT, PACKED>(S, A, e >> 8, (int)(e & 255u), rc);
                }
            }
            __syncwarp();  // tables are rewritten by the next chunk
        }

        // ---- flush the staged survivors: one global atomic per warp-tile
        const unsigned int staged = min(S.stage_count, (unsigned)SW_STAGE);
        if (EMIT == 1 && A.go.cnt) {  // events straight into their post-pass groups
            for (unsigned int i = lane; i < staged; i += 32) {
                const EventRec ev = S.stage[i];
                const uint64_t pos = A.go.place(ev.hash, A.g_count, A.cap);
                if (pos == ~0ull) continue;
                reinterpret_cast<EventRec *>(A.out)[pos] = ev;
                if (ev.recflag & EV_PENDING) A.pend[atomicAdd(A.g_pend, 1ull)] = (uint32_t)pos;
            }
        } else if (staged) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(A.g_count, (unsigned long long)staged);
            base = __shfl_sync(0xffffffffu, base, 0);
            for (unsigned int i = lane; i < staged; i += 32) {
                if (base + i >= A.cap) continue;
                if (EMIT == 0) reinterpret_cast<syl_survivor *>(A.out)[base + i] = reinterpret_cast<const syl_survivor *>(S.stage)[i];
                else {
                    const EventRec ev = S.stage[i];
                    reinterpret_cast<EventRec *>(A.out)[base + i] = ev;
                    if (ev.recflag & EV_PENDING) A.pend[atomicAdd(A.g_pend, 1ull)] = (uint32_t)(base + i);
                }
            }
        }
        __syncwarp();
        t = tn;
    }
}

using seedw_kern_t = void (*)(const SeedWArgs);

#define SEEDW_DEFINE_KERNELS(NAME, K, EMIT, PACKED)                  \
    seedw_kern_t NAME(int W) {                                       \
        switch (W) {                                                 \
            case 24: return k_seed_w<K, 0, EMIT, 24, PACKED>;        \
            case 30: return k_seed_w<K, 0, EMIT, 30, PACKED>;        \
            default: return k_seed_w<K, 0, EMIT, 32, PACKED>;        \
        }                                                            \
    }

seedw_kern_t seedw_kernels_k31_sv(int W);
seedw_kern_t seedw_kernels_k31_ev(int W);
seedw_kern_t seedw_kernels_k21_sv(int W);
seedw_kern_t seedw_kernels_k21_ev(int W);
seedw_kern_t seedw_kernels_k31_sv_p(int W);
seedw_kern_t seedw_kernels_k31_ev_p(int W);
seedw_kern_t seedw_kernels_k21_sv_p(int W);
seedw_kern_t seedw_kernels_k21_ev_p(int W);

template <bool PACKED>
constexpr size_t seedw_smem_bytes() { return 1024 + (size_t)SW_WARPS * sizeof(SeedWSlab<PACKED>); }

}  // namespace syl
