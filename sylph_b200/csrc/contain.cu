// contain.cu — containment query / profile on sm_90a.
//
// Replaces, for every (sample, genome) pair at once, the get_stats loops of contain()
// (src/contain.rs:284-292 pass 1, :297-327 pass 2) including
//   probe loop                      src/contain.rs:632-652
//   median / Poisson cut / means    :657-690   (statrs Poisson CDF -> 29-entry cutoff table)
//   ratio_lambda                    src/inference.rs:207-242
//   ani_from_lambda                 src/contain.rs:817-847
//   bootstrap_interval              :849-898   (fastrand WyRand, counter-based here)
//   winner_table + pass-2 lost rule :410-430, :641-646
//   derep_if_reassign_threshold     :353-375 and abundances :319-326 (host side of syl_profile)
//
// Formulation.  The reference probes the sample's hash map with every k-mer of every genome
// (|DB| probes per sample).  |sample| (~10^6) << |DB| (~10^8..10^9), so the join is turned
// around: all database k-mers (genome_kmers and tracked) are sorted ONCE into a global index
// (key -> genome); each sample key then looks itself up through a bucket directory
// (keys are uniform hashes, so bucket = mulhi(key, M) is a perfect interpolation) and walks
// the equal range.  Work per sample = |sample| short probes + #hits, independent of how many
// genomes the database holds, and the database is never streamed.  The per-genome statistics
// are functions of the multiset of hit counts: the join accumulates a 256-bin histogram of the
// counts per (sample, genome) pair and one warp per pair derives everything from it (a count
// >= 256 anywhere, or histograms beyond 8 GB, send the call through the CSR formulation instead:
// count, scan, scatter, exact radix select for the median — no range limit).  In pass 2 the
// winner of a k-mer is the pass-1 survivor that comes first in its sample's order (ANI
// descending, genome ascending) inside that k-mer's equal range — a purely local decision, so no
// global k-mer -> winner map is ever materialised.  Both formulations run through one staged
// driver (contain_fast below).
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <functional>
#include <new>
#include <vector>

#include "contain.hpp"
#include "crmath.cuh"
#include "scan_plan.hpp"

namespace syl {

// src/contain.rs:664-675 with src/constants.rs:3: largest cov with PoissonCDF(cov; m) < 0.9999999999
// for integer medians m = 1..29 (statrs 0.16.1 cdf = Q(cov+1, m)); index 0 unused.
__constant__ uint32_t c_pois_cut[30] = {0,  11, 15, 18, 21, 24, 26, 28, 31, 33, 35, 37, 39, 41, 43,
                                        45, 46, 48, 50, 52, 53, 55, 57, 58, 60, 62, 63, 65, 67, 68};

struct StatParams {
    int k;
    int no_ci, no_adj, mean_coverage;
    double min_number_kmers, min_count_correct, min_ani;
};

// Extras of the device-driven profile (contain_fast below): pass 1 records the containment count of every
// emitted row in a dense table; pass 2 stashes it (and the genome size) in the row for the host-side
// derep / abundance step, which then needs nothing but the rows.
struct StatExtra {
    uint32_t *contain1_out = nullptr;       // [S x G], pass 1
    const uint32_t *contain1_in = nullptr;  // [S x G], pass 2 -> row.reserved
    const uint64_t *gn_size = nullptr;      // [G], pass 2 -> row.seq_abund
    uint64_t pair_stride = 0;               // G
};

// ---- per-genome statistics: one warp per genome ---------------------------------------------

struct RatioOut { bool ok; double lambda; };

// src/inference.rs:207-242 on a histogram H[1..16] of the non-zero values (H[v] = #values == v),
// nz = number of non-zero values in full_covs.
__device__ __forceinline__ RatioOut ratio_lambda_hist(const uint32_t *H, uint32_t nz, double min_count_correct) {
    RatioOut r = {false, 0.0};
    uint32_t distinct = 0, mode = 0, best = 0;
    for (uint32_t v = 1; v <= 16; v++) {
        if (H[v]) distinct++;
        if (H[v] && H[v] >= best) { best = H[v]; mode = v; }  // ties -> larger value (:226-230)
    }
    if (distinct == 1) return r;                  // :221-223
    if (nz < 25u) return r;                       // SAMPLE_SIZE_CUTOFF
    if (mode == 0 || mode >= 16 || H[mode + 1] == 0) return r;
    const double cp1 = (double)H[mode + 1], cm = (double)H[mode];
    if (cp1 < min_count_correct || cm < min_count_correct) return r;
    r.ok = true;
    r.lambda = cp1 / cm * (double)(mode + 1);
    return r;
}

// src/contain.rs:817-847.  pow and exp correctly rounded (crmath.cuh): the ANI decides the -m gate and the winner
// order, where CUDA's last bit and the reference's glibc last bit would print different rows.
__device__ __forceinline__ bool ani_from_lambda_dev(double lambda, double k, uint64_t nz, uint64_t nfull, double *out) {
    const double adj = (double)nz / (1. - crm::cr_exp(-lambda)) / (double)nfull;
    const double ani = crm::cr_pow(adj, 1. / k);
    if (ani < 0. || isnan(ani)) return false;
    *out = ani;
    return true;
}

// Everything get_stats derives from (n hits, median, sum and count of the kept coverages, histogram of
// the kept values 1..16) for one (sample, genome) pair; one lane.  src/contain.rs:690-814.
__device__ __forceinline__ void stats_emit(uint32_t sample_idx, uint64_t g, uint32_t n, uint32_t gl, uint32_t median, uint32_t sum,
                                           uint32_t nz, const uint32_t *hist, const uint32_t *lost, uint32_t genome_base,
                                           const StatParams &P, int pass2, syl_ani_row *__restrict__ rows, uint64_t rows_cap,
                                           uint32_t *__restrict__ boot_rows, uint32_t *__restrict__ hist_out, uint64_t boot_cap,
                                           unsigned long long *__restrict__ n_rows, unsigned long long *__restrict__ n_boot,
                                           const StatExtra X = StatExtra()) {
    const double k = (double)P.k;
    const uint64_t nfull = (uint64_t)(gl - n) + nz;
    const double naive_ani = crm::cr_pow((double)n / (double)gl, 1. / k);
    const double geq1_mean = (double)sum / (double)n;  // :690 divides by covs.len()
    uint32_t status;
    double lam = 0.;
    if ((double)median > 2.) {
        status = SYL_LAMBDA_HIGH;
    } else {
        RatioOut r = ratio_lambda_hist(hist, nz, P.min_count_correct);
        status = r.ok ? SYL_LAMBDA_VALUE : SYL_LAMBDA_LOW;
        lam = r.lambda;
    }
    double final_cov;
    if (status == SYL_LAMBDA_VALUE) final_cov = lam;
    else if ((double)median < 15.) final_cov = geq1_mean;
    else final_cov = P.mean_coverage ? geq1_mean : (double)median;
    double est = 0.;
    const bool has_lambda = status == SYL_LAMBDA_VALUE;
    const bool has_est = has_lambda && ani_from_lambda_dev(final_cov, k, nz, nfull, &est);
    const double final_ani = (!has_lambda || !has_est || P.no_adj) ? naive_ani : est;
    if (final_ani < P.min_ani) return;  // :746-764

    syl_ani_row r;
    r.sample = sample_idx;
    r.genome = genome_base + (uint32_t)g;
    r.lambda_status = status;
    r.ci_valid = 0;
    r.contain = n;
    r.glen = gl;
    r.kmers_lost = pass2 ? (int64_t)lost[g] : -1;
    r.naive_ani = naive_ani;
    r.final_est_ani = final_ani;
    r.final_est_cov = final_cov;
    r.mean_cov = geq1_mean;
    r.median_cov = (double)median;
    r.lambda = has_lambda ? lam : 0.;
    r.ci[0] = r.ci[1] = r.ci[2] = r.ci[3] = 0.;
    r.rel_abund = 0.;
    r.seq_abund = X.gn_size ? (double)X.gn_size[g] : 0.;
    r.reserved = X.contain1_in ? (double)X.contain1_in[(uint64_t)sample_idx * X.pair_stride + g] : 0.;
    if (X.contain1_out) X.contain1_out[(uint64_t)sample_idx * X.pair_stride + g] = n;
    const unsigned long long ri = atomicAdd(n_rows, 1ull);  // compact output; the host orders rows
    if (ri >= rows_cap) return;
    rows[ri] = r;
    if (!P.no_ci && has_lambda) {
        const unsigned long long bi = atomicAdd(n_boot, 1ull);
        if (bi < boot_cap) {
            boot_rows[bi] = (uint32_t)ri;
            for (int v = 0; v < 17; v++) hist_out[bi * 17 + v] = v == 0 ? (uint32_t)(gl - n) : hist[v];
        }
    }
}

constexpr int STAT_WARPS = 4;

// CSR formulation: one warp per (sample, genome) over the pair's hit values covs[off[pair], off[pair] + cnt[pair])
__global__ void __launch_bounds__(STAT_WARPS * 32)
k_stats(const uint32_t *__restrict__ cnt, const uint64_t *__restrict__ off, const uint32_t *__restrict__ covs,
        const uint32_t *__restrict__ glen, const uint32_t *__restrict__ lost, uint64_t n_genomes, uint64_t n_pairs,
        uint32_t genome_base, StatParams P, int pass2, syl_ani_row *__restrict__ rows, uint64_t rows_cap,
        uint32_t *__restrict__ boot_rows, uint32_t *__restrict__ hist_out, uint64_t boot_cap,
        unsigned long long *__restrict__ n_rows, unsigned long long *__restrict__ n_boot, const StatExtra X) {
    __shared__ uint32_t s_hist[STAT_WARPS][256];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint64_t pair = (uint64_t)blockIdx.x * STAT_WARPS + w;
    if (pair >= n_pairs) return;
    const uint32_t sample_idx = (uint32_t)(pair / n_genomes);
    const uint64_t g = pair - (uint64_t)sample_idx * n_genomes;
    uint32_t *hist = s_hist[w];
    cnt += (uint64_t)sample_idx * n_genomes;
    off += (uint64_t)sample_idx * n_genomes;
    if (lost) lost += (uint64_t)sample_idx * n_genomes;
    const uint32_t n = cnt[g];
    const uint32_t gl = glen[g];
    if (n == 0) return;                                   // covs.is_empty() :654
    if ((double)gl < P.min_number_kmers) return;          // :627
    const uint32_t *cv = covs + off[g];

    // exact median = element of rank n/2 (0-based) by MSB-first radix select
    uint32_t prefix = 0, kth = n / 2;
    for (int pass = 3; pass >= 0; pass--) {
        for (int b = lane; b < 256; b += 32) hist[b] = 0;
        __syncwarp();
        const uint32_t hi_mask = pass == 3 ? 0u : (0xFFFFFFFFu << (8 * (pass + 1)));
        for (uint32_t i = lane; i < n; i += 32) {
            const uint32_t v = cv[i];
            if ((v & hi_mask) == prefix) atomicAdd(&hist[(v >> (8 * pass)) & 255u], 1u);
        }
        __syncwarp();
        // lane l owns bins [8l, 8l+8)
        uint32_t local[8], tot = 0;
#pragma unroll
        for (int q = 0; q < 8; q++) { local[q] = hist[8 * lane + q]; tot += local[q]; }
        uint32_t incl = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        const uint32_t excl = incl - tot;
        const bool mine = kth >= excl && kth < incl;
        uint32_t digit = 0, newk = 0;
        if (mine) {
            uint32_t acc = excl;
#pragma unroll
            for (int q = 0; q < 8; q++) {
                if (kth >= acc && kth < acc + local[q]) { digit = 8 * lane + q; newk = kth - acc; }
                acc += local[q];
            }
        }
        const uint32_t src = __ffs(__ballot_sync(0xffffffffu, mine)) - 1;
        digit = __shfl_sync(0xffffffffu, digit, src);
        kth = __shfl_sync(0xffffffffu, newk, src);
        prefix |= digit << (8 * pass);
        __syncwarp();
    }
    const uint32_t median = prefix;
    const uint32_t max_cov = median < 30u ? c_pois_cut[median] : 0xFFFFFFFFu;  // f64::MAX

    // sums over full_covs = zeros ++ {cov <= max_cov}; small histogram for ratio_lambda
    for (int b = lane; b < 32; b += 32) hist[b] = 0;
    __syncwarp();
    uint32_t sum = 0, nz = 0;  // u32 sum wraps like iter().sum::<u32>() in a release build
    const bool want_hist = median <= 2u;
    for (uint32_t i = lane; i < n; i += 32) {
        const uint32_t v = cv[i];
        if (v <= max_cov) {
            sum += v;
            nz++;
            if (want_hist && v <= 16u) atomicAdd(&hist[v], 1u);
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, d);
        nz += __shfl_xor_sync(0xffffffffu, nz, d);
    }
    __syncwarp();
    if (lane != 0) return;

    stats_emit(sample_idx, g, n, gl, median, sum, nz, hist, lost, genome_base, P, pass2, rows, rows_cap, boot_rows, hist_out,
               boot_cap, n_rows, n_boot, X);
}


// ---- histogram formulation of one get_stats pass ------------------------------------------------
// get_stats only needs, per (sample, genome), the multiset of the hit k-mers' sample counts: its
// median, the sum / number of the values below the Poisson cut-off and how many are 1, 2, .., 16.
// All of that follows from a histogram of the values, which the join can accumulate directly:
// ONE probe pass per get_stats pass (the CSR formulation probes twice: count, then fill) and a
// k_stats that reads 1 KB per pair instead of selecting a median from a value list.  Values
// >= COV_BINS (a genome covered 256x or deeper) are only counted in `ovf`; if there are any, the
// call is redone in the CSR formulation.

// ---- thread -> (sample, key) mapping of the join kernels ---------------------------------------------------------
// Plain form (rb == nullptr): grid (key blocks, samples), one key per thread.  With several samples that order walks
// the db index once PER SAMPLE (the blocks of sample s+1 start when sample s is through), and the index is far larger
// than L2: 16 samples cost 16x the DRAM traffic of one.  Tiled form: the hash space is cut into R ranges of equal
// db-bucket count and the block index runs sample-fastest over (range, sample), so the blocks resident at any time
// probe the SAME stretch of the index for all samples and that stretch comes from DRAM once.  rb[s * (R+1) + r] =
// index of sample s's first key in range r (k_range_bounds); a block loops over its range's keys (~100).
struct KeyMap { const uint32_t *rb; uint32_t R, S; };

template <class F>
__device__ __forceinline__ void for_each_key(const KeyMap km, const SampleView *__restrict__ views, F body) {
    if (!km.rb) {
        const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
        if (i < views[blockIdx.y].n) body((uint32_t)blockIdx.y, i);
        return;
    }
    const uint32_t s = blockIdx.x % km.S, r = blockIdx.x / km.S;
    const uint32_t *b = km.rb + (uint64_t)s * (km.R + 1) + r;
    const uint32_t lo = b[0], hi = b[1];
    for (uint64_t i = (uint64_t)lo + threadIdx.x; i < hi; i += blockDim.x) body(s, i);
}

__global__ void k_range_bounds(const SampleView *__restrict__ views, uint32_t S, uint32_t R, uint64_t bpr, uint64_t M, uint64_t NB,
                               uint32_t *__restrict__ rb) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)S * (R + 1)) return;
    const uint32_t s = (uint32_t)(t / (R + 1)), r = (uint32_t)(t % (R + 1));
    const SampleView sv = views[s];
    const uint64_t want = (uint64_t)r * bpr;  // first key whose bucket is >= want (buckets are monotone in the key)
    uint64_t lo = 0, hi = sv.n;
    if (r == R) lo = sv.n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (bucket_of(sv.hash[mid], M, NB) < want) lo = mid + 1; else hi = mid;
    }
    rb[t] = (uint32_t)lo;
}

// f(g) for the genome index g of every entry of one k-mer's equal range [lo, e) of the db index.  Tracked entries
// only take part in pass 2's winner decision, so they are skipped unless TRACKED.  The genome ids are loaded four at
// a time: a long range walked one dependent load at a time holds its whole warp for range x DRAM latency.
template <bool TRACKED = false, class F>
__device__ __forceinline__ void walk_range(const uint32_t *__restrict__ gid, uint32_t lo, uint32_t e, F f) {
    for (uint32_t j = lo; j < e; j += 4) {
        uint32_t gq[4];
#pragma unroll
        for (int q = 0; q < 4; q++) gq[q] = j + q < e ? gid[j + q] : 0xFFFFFFFFu;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (j + q >= e) continue;
            if (!TRACKED && (gq[q] & 1u)) continue;
            f(gq[q] >> 1);
        }
    }
}

// What a walk produces: count histograms (JOIN_HIST), or the CSR formulation's count walk (cnt) or fill walk (covs).
enum JoinOut { JOIN_HIST, JOIN_CSR_COUNT, JOIN_CSR_FILL };

// Where the hits of a walk go, per (sample, genome) pair.  Histogram formulation: touched and the count histograms,
// values >= COV_BINS only counted in ovf.  CSR formulation: the count walk adds up the hits per pair in cnt; after
// the scan of cnt into off, the fill walk writes each hit's sample count to covs[off[pair] + cursor[pair]++].
struct PairOut {
    uint8_t *touched; uint32_t *chist; unsigned long long *ovf;
    uint32_t *cnt; const uint64_t *off; uint32_t *cursor; uint32_t *covs;

    template <JoinOut OUT>
    __device__ __forceinline__ void hit(uint64_t pair, uint32_t c) const {
        if (OUT == JOIN_CSR_COUNT) { atomicAdd(&cnt[pair], 1u); return; }
        if (OUT == JOIN_CSR_FILL) { covs[off[pair] + atomicAdd(&cursor[pair], 1u)] = c; return; }
        // no per-genome hit counter: the sample's k-mers concentrate on the few genomes that are
        // present, and a million atomics on a handful of adjacent counters serialise in one L2
        // slice (measured: 2/3 of the pass-1 join's time).  The hit count is the histogram's total.
        if (!touched[pair]) touched[pair] = 1;
        if (c < COV_BINS) atomicAdd(&chist[pair * COV_BINS + c], 1u);
        else atomicAdd(ovf, 1ull);
    }
};

// Pass-1 probe: every sample key looks up its equal range in the db index and records it in `hits` (for pass 2 and,
// in the CSR formulation, for pass 1's count / fill walks).  PROBE_ONLY == false also accumulates the count histograms.
template <bool PROBE_ONLY>
__global__ void k_join_hist(const SampleView *__restrict__ views, uint64_t G,
                            const uint64_t *__restrict__ keys, const uint32_t *__restrict__ gid, uint64_t N,
                            const uint32_t *__restrict__ bstart, uint64_t M, uint64_t NB, uint64_t maxkey,
                            const PairOut out, uint2 *__restrict__ hits, uint64_t hits_stride, const KeyMap km) {
  for_each_key(km, views, [&](const uint32_t smp, const uint64_t i) {
    const SampleView sv = views[smp];
    const uint64_t key = sv.hash[i];
    const uint32_t c = sv.count[i];
    if (key > maxkey || c == 0) return;  // count 0: src/contain.rs:634-636
    const uint64_t b = bucket_of(key, M, NB);
    uint32_t lo = bstart[b];
    const uint32_t hi = bstart[b + 1];
    // A k-mer shared by many genomes has a long equal range, and a thread walking it one dependent
    // load at a time holds its whole warp for range x DRAM latency.  Keys and genome ids are
    // therefore fetched four at a time (independent loads; reads past the bucket stay inside the
    // arrays, which hold N entries).
    const uint32_t n4 = (uint32_t)N;
    for (;;) {  // first position with keys[lo] >= key
        if (lo >= hi) return;  // (hits is zero-filled by the caller)
        uint64_t kq[4];
#pragma unroll
        for (int q = 0; q < 4; q++) kq[q] = lo + q < n4 ? keys[lo + q] : 0xFFFFFFFFFFFFFFFFull;
        int adv = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) adv += (lo + q < hi && kq[q] < key) ? 1 : 0;  // keys ascend: a prefix
        lo += adv;
        if (adv < 4) break;
    }
    if (lo >= hi || keys[lo] != key) return;
    uint32_t e = lo;  // end of the equal range
    for (;;) {
        uint64_t kq[4];
#pragma unroll
        for (int q = 0; q < 4; q++) kq[q] = e + q < n4 ? keys[e + q] : 0xFFFFFFFFFFFFFFFFull;
        int adv = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) adv += (e + q < hi && kq[q] == key) ? 1 : 0;
        e += adv;
        if (adv < 4) break;
    }
    if (hits) hits[(uint64_t)smp * hits_stride + i] = make_uint2(lo, e - lo);  // equal range in the db
    if (!PROBE_ONLY) {
        const uint64_t row = (uint64_t)smp * G;
        walk_range(gid, lo, e, [&](const uint32_t g) { out.hit<JOIN_HIST>(row + g, c); });
    }
  });
}

// ---- scan formulation of pass 1 (the join the reference does, src/contain.rs:632-652) ---------------------------------
// For a call of few samples against a database in host memory, building the index costs far more than the joins.  The
// scan streams the genome k-mers of a chunk of whole genomes instead, and each one probes every sample's lookup table
// (scan_plan.hpp): the same (sample key, genome k-mer) hits as the index join, so the same per-pair outputs.

// tables[s].M, and the directory of an empty sample
__global__ void k_table_params(SampleTable *__restrict__ tables, uint32_t S) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    SampleTable &t = tables[s];
    t.M = table_mult(t.n ? t.hash[t.n - 1] : 0, t.NB);
    if (!t.n) { const_cast<uint32_t *>(t.dir)[0] = 0; const_cast<uint32_t *>(t.dir)[1] = 0; }
}

// grid (key blocks, samples s0 ..): fingerprints and directory entries of every key
__global__ void k_table_fill(const SampleTable *__restrict__ tables, uint32_t s0) {
    const SampleTable t = tables[s0 + blockIdx.y];
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.n) return;
    const_cast<uint32_t *>(t.fp)[i] = (uint32_t)t.hash[i];
    table_dir_entries(t.hash, t.n, i, t.M, t.NB, const_cast<uint32_t *>(t.dir));
}

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_PER_THREAD = 4;  // k-mers per thread: two 128-bit loads, four independent probe chains per sample

// One thread per SCAN_PER_THREAD consecutive k-mers of the chunk (coalesced 128-bit loads).  A k-mer's genome is the last
// g with off[g] <= its index (empty genomes share their successor's offset).  Every k-mer probes every sample's table;
// a hit with a non-zero count (src/contain.rs:634-636) goes to pair (s, g) as in the index join.
template <JoinOut OUT>
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan(const ScanChunk ch, uint32_t S, uint64_t G, const PairOut out) {
    const uint64_t i0 = ((uint64_t)blockIdx.x * SCAN_THREADS + threadIdx.x) * SCAN_PER_THREAD;
    if (i0 >= ch.n) return;
    uint64_t kq[SCAN_PER_THREAD];
    const int nk = ch.n - i0 < SCAN_PER_THREAD ? (int)(ch.n - i0) : SCAN_PER_THREAD;
    if (nk == SCAN_PER_THREAD) {
        const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(ch.kmers + i0);
        const ulonglong2 a = p[0], b = p[1];
        kq[0] = a.x; kq[1] = a.y; kq[2] = b.x; kq[3] = b.y;
    } else {
#pragma unroll
        for (int q = 0; q < SCAN_PER_THREAD; q++) kq[q] = q < nk ? ch.kmers[i0 + q] : 0;
    }
    uint64_t lo = 0, hi = G;  // off[lo] <= i0 < off[hi]
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) >> 1;
        if (ch.off[mid] <= i0) lo = mid; else hi = mid;
    }
    uint32_t g[SCAN_PER_THREAD];
#pragma unroll
    for (int q = 0; q < SCAN_PER_THREAD; q++) {
        if (q < nk) while (ch.off[lo + 1] <= i0 + q) lo++;
        g[q] = (uint32_t)lo;
    }
    for (uint32_t s = 0; s < S; s++) {
        const SampleTable t = ch.tables[s];
        const uint64_t row = (uint64_t)s * G;
        uint32_t b0[SCAN_PER_THREAD], b1[SCAN_PER_THREAD];
#pragma unroll
        for (int q = 0; q < SCAN_PER_THREAD; q++) {
            const uint64_t b = table_bucket(kq[q], t.M, t.NB);
            b0[q] = q < nk ? t.dir[b] : 0;
            b1[q] = q < nk ? t.dir[b + 1] : 0;
        }
#pragma unroll
        for (int q = 0; q < SCAN_PER_THREAD; q++) {
            for (uint32_t j = b0[q]; j < b1[q]; j++) {
                if (t.fp[j] != (uint32_t)kq[q] || t.hash[j] != kq[q]) continue;
                const uint32_t c = t.count[j];
                if (c) out.hit<OUT>(row + g[q], c);
            }
        }
    }
}

int build_tables(syl_ctx *ctx, const SampleView *views, uint32_t S, DevBuf<SampleTable> &tables, DevBuf<uint32_t> &dir,
                 DevBuf<uint32_t> &fp, std::vector<SampleTable> &h) {
    cudaStream_t st = ctx->stream;
    uint64_t nd = 0, nf = 0, max_n = 0;
    for (uint32_t s = 0; s < S; s++) {
        nd += table_buckets(views[s].n) + 1;
        nf += views[s].n;
        max_n = std::max(max_n, views[s].n);
    }
    SYL_TRY(tables.alloc(S, st)); SYL_TRY(dir.alloc(nd, st)); SYL_TRY(fp.alloc(nf, st));
    h.resize(S);
    nd = nf = 0;
    for (uint32_t s = 0; s < S; s++) {
        const uint64_t NB = table_buckets(views[s].n);
        h[s] = SampleTable{views[s].hash, views[s].count, fp.p + nf, dir.p + nd, views[s].n, NB, 0};
        nd += NB + 1;
        nf += views[s].n;
    }
    if (!S) return SYL_OK;
    // a pageable source is staged by the driver before cudaMemcpyAsync returns
    SYL_CUDA(cudaMemcpyAsync(tables.p, h.data(), S * sizeof(SampleTable), cudaMemcpyHostToDevice, st));
    KernelTimer kt(ctx, SYL_KERNEL_SCAN);
    k_table_params<<<nblk(S, 128), 128, 0, st>>>(tables.p, S);
    ctx->launches++;
    for (uint32_t s0 = 0; s0 < S && max_n; s0 += 65535) {
        k_table_fill<<<dim3(nblk(max_n, 256), std::min<uint32_t>(S - s0, 65535)), 256, 0, st>>>(tables.p, s0);
        ctx->launches++;
    }
    SYL_CUDA(cudaGetLastError());
    return SYL_OK;
}

// one warp per (sample, genome); lane l owns the bins [8l, 8l+8)
__global__ void __launch_bounds__(STAT_WARPS * 32)
k_stats_hist(const uint8_t *__restrict__ touched, const uint32_t *__restrict__ chist,
             const uint32_t *__restrict__ glen, const uint32_t *__restrict__ lost, uint64_t n_genomes, uint64_t n_pairs,
             uint32_t genome_base, StatParams P, int pass2, syl_ani_row *__restrict__ rows, uint64_t rows_cap,
             uint32_t *__restrict__ boot_rows, uint32_t *__restrict__ hist_out, uint64_t boot_cap,
             unsigned long long *__restrict__ n_rows, unsigned long long *__restrict__ n_boot, const StatExtra X = StatExtra()) {
    __shared__ uint32_t s_hist[STAT_WARPS][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint64_t pair = (uint64_t)blockIdx.x * STAT_WARPS + w;
    if (pair >= n_pairs) return;
    const uint32_t sample_idx = (uint32_t)(pair / n_genomes);
    const uint64_t g = pair - (uint64_t)sample_idx * n_genomes;
    if (!touched[pair]) return;                           // covs.is_empty() :654
    const uint32_t gl = glen[g];
    if ((double)gl < P.min_number_kmers) return;          // :627
    if (lost) lost += (uint64_t)sample_idx * n_genomes;
    const uint4 *hp = reinterpret_cast<const uint4 *>(chist + pair * COV_BINS + 8 * lane);
    const uint4 h0 = hp[0], h1 = hp[1];
    const uint32_t h[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    uint32_t tot = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) tot += h[q];
    uint32_t incl = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    const uint32_t n = __shfl_sync(0xffffffffu, incl, 31);  // number of hit k-mers
    // median = value of rank n/2 (0-based) in ascending order (:659-660)
    const uint32_t kth = n / 2, excl = incl - tot;
    uint32_t med = 0;
    if (kth >= excl && kth < incl) {
        uint32_t acc = excl;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            if (kth >= acc && kth < acc + h[q]) med = 8 * lane + q;
            acc += h[q];
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) med |= __shfl_xor_sync(0xffffffffu, med, d);  // exactly one lane holds it
    const uint32_t median = med;
    const uint32_t max_cov = median < 30u ? c_pois_cut[median] : 0xFFFFFFFFu;  // f64::MAX
    uint32_t sum = 0, nz = 0;  // u32 sum wraps like iter().sum::<u32>() in a release build
    uint32_t *hist = s_hist[w];
    hist[lane] = 0;
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const uint32_t v = 8 * lane + q;
        if (v <= max_cov) {
            sum += v * h[q];
            nz += h[q];
            if (v >= 1 && v <= 16u) hist[v] = h[q];
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, d);
        nz += __shfl_xor_sync(0xffffffffu, nz, d);
    }
    __syncwarp();
    if (lane != 0) return;
    stats_emit(sample_idx, g, n, gl, median, sum, nz, hist, lost, genome_base, P, pass2, rows, rows_cap, boot_rows, hist_out,
               boot_cap, n_rows, n_boot, X);
}

// ---- bootstrap (src/contain.rs:849-898) -------------------------------------------------------
// fastrand 2.1.1 WyRand: state after d draws = seed + d*C0, so draw d is random access.
__device__ __forceinline__ uint64_t wyrand_at(uint64_t seed, uint64_t d) {
    const uint64_t s = seed + d * 0x2d358dccaa6c78a5ull;
    const uint64_t t = s ^ 0x8bb84b93962eacc9ull;
    return (s * t) ^ __umul64hi(s, t);
}

constexpr int BOOT_THREADS = 256;

// 64 x 64 -> 128-bit product, xor of the two halves (WyRand's output function).  The 128-bit type
// compiles to four IMAD.WIDE with carry-in/out (11 instructions with the xors); a hand-split into
// 32-bit halves costs 18 because every 64-bit addend needs an aligned register pair.
__device__ __forceinline__ uint64_t mum_xor(uint64_t a, uint64_t b) {
    const unsigned __int128 p = (unsigned __int128)a * b;
    return (uint64_t)p ^ (uint64_t)(p >> 64);
}

// ctr += (x >= t) for t >= 1, given nt = 2^64 - t: the carry out of the 64-bit sum x + nt.
// Three instructions (IADD3 carry-out, IADD3.X, add-with-carry); the C forms compile to 5-6.
__device__ __forceinline__ void count_ge(uint32_t &ctr, uint64_t x, uint64_t nt) {
    asm("{\n\t.reg .u32 d;\n\tadd.cc.u32 d, %1, %3;\n\taddc.cc.u32 d, %2, %4;\n\taddc.u32 %0, %0, 0;\n\t}"
        : "+r"(ctr) : "r"((uint32_t)x), "r"((uint32_t)(x >> 32)), "r"((uint32_t)nt), "r"((uint32_t)(nt >> 32)));
}

// Smallest 64-bit draw x whose Lemire index floor(x*n / 2^64) reaches c, for 0 <= c < n < 2^32:
// ceil(c * 2^64 / n) by two 64/32 long-division steps.  c >= n has no such draw (callers mask it).
__device__ __forceinline__ uint64_t lemire_threshold(uint64_t c, uint64_t n) {
    if (c >= n) return ~0ull;
    const uint64_t d1 = c << 32, q1 = d1 / n, r1 = d1 % n;
    const uint64_t d0 = r1 << 32, q0 = d0 / n, r0 = d0 % n;
    return (q1 << 32) + q0 + (r0 ? 1 : 0);
}

// One CTA resamples |full| values for one iteration `it` of one bootstrapped row.
// H layout per row: [0] = number of zeros, [v] = #values == v (v = 1..16; all values of a
// bootstrapped row are <= 15 because its median is <= 2).  ratio_lambda / ani_from_lambda only
// need the histogram of the NON-ZERO resampled values and the total, so zero draws (the large
// majority) cost nothing beyond the RNG.
__device__ __forceinline__ void boot_one(uint32_t row, uint32_t it, const uint32_t *__restrict__ hist_in, const StatParams &P,
                                         double *__restrict__ res_ani, double *__restrict__ res_lambda, uint8_t *__restrict__ res_ok,
                                         uint32_t *__restrict__ reject_flag, uint32_t *Hb, uint64_t *cum, uint64_t *thr, uint64_t *nthr) {
    const uint32_t *H = hist_in + (uint64_t)row * 17;
    if (threadIdx.x < 17) Hb[threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        uint64_t acc = 0;
        for (int v = 0; v < 17; v++) { acc += H[v]; cum[v] = acc; }  // cum[v] = #values <= v
    }
    __syncthreads();
    if (threadIdx.x < 16) {
        const uint64_t t = lemire_threshold(cum[threadIdx.x], cum[16]);
        thr[threadIdx.x] = t;
        nthr[threadIdx.x] = 0ull - t;
    }
    __syncthreads();
    const uint64_t n = cum[16];
    const uint32_t n32 = (uint32_t)n;  // |full| = |genome_kmers| < 2^32
    // Lemire's index is hi = floor(x*n / 2^64), and hi >= c  <=>  x >= ceil(c * 2^64 / n): the four
    // common class boundaries are compared on the 64-bit draw itself, so the two 32x32->64 multiplies
    // of the index are only paid by the rare draws that need it (values >= 4, rejection candidates).
    const uint64_t t3 = thr[3], nt0 = 0ull - thr[0], nt1 = 0ull - thr[1], nt2 = 0ull - thr[2], nt3 = 0ull - t3;
    uint32_t ge[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // ge[v] = draws with a value > v (x >= thr[v])
    const bool more_than_3 = cum[3] < n, more_than_7 = cum[7] < n;
    // no value above 3: the branch below is never wanted; an all-ones boundary does that without a second test in the
    // loop (a draw of exactly 2^64-1 would still enter, harmlessly: every count it touches is zeroed after the loop)
    const uint64_t t3_eff = more_than_3 ? t3 : ~0ull;
    uint32_t vmax = 8;  // largest value present (cum[vmax] = n): no draw lies at or above boundary vmax
    while (vmax < 16 && cum[vmax] < n) vmax++;
    // draw number d = it*n + j + 1; WyRand state s(d) = 7 + d*C0, advanced by BOOT_THREADS*C0 per trip
    uint64_t s = 7ull + ((uint64_t)it * n + threadIdx.x + 1) * 0x2d358dccaa6c78a5ull;
    const uint64_t s_step = (uint64_t)BOOT_THREADS * 0x2d358dccaa6c78a5ull;
    for (uint32_t j = threadIdx.x; j < n32; j += BOOT_THREADS, s += s_step) {
        const uint64_t x = mum_xor(s, s ^ 0x8bb84b93962eacc9ull);
        // fastrand gen_mod_u64 redraws when lo = (x*n) mod 2^64 < (2^64 - n) mod n.  lo < n < 2^32 needs
        // the low word of x_lo*n to be < n (probability n / 2^32): only then is lo formed.  The empty volatile asm
        // pins that to the branch (otherwise the full product is hoisted into the loop: 9 instructions per draw, not 3).
        if ((uint32_t)x * n32 < n32) {
            uint64_t xr = x;
            asm volatile("" : "+l"(xr));
            const uint64_t lo = xr * n;
            if (lo < n && lo < (0ull - n) % n) atomicExch(reject_flag + row, 1u);  // the reference would redraw
        }
        // full_covs[hi] = v with cum[v-1] <= hi < cum[v].  Branch-free for the common values (0: most draws;
        // 1, 2, 3: counted in registers) — lanes of a warp draw different values, a branch per value would
        // serialise them (measured: 60 instructions per draw with the branches, 23 of 32 lanes active).
        count_ge(ge[0], x, nt0);
        count_ge(ge[1], x, nt1);
        count_ge(ge[2], x, nt2);
        count_ge(ge[3], x, nt3);
        if (x >= t3_eff) {
            // a value >= 4: a few percent of the draws of a row with median 2, but then a third of the WARPS have
            // such a lane.  Values 4..7 are counted like 0..3 (negated boundaries from shared memory); beyond 7
            // the remaining boundaries are walked upwards (rare).
            count_ge(ge[4], x, nthr[4]);
            count_ge(ge[5], x, nthr[5]);
            count_ge(ge[6], x, nthr[6]);
            if (more_than_7 && x >= thr[7]) {
                ge[7]++;
                uint32_t v = 8;
                while (v < vmax && x >= thr[v]) v++;
                atomicAdd(&Hb[v], 1u);
            }
        }
    }
    // a boundary of 0 has every draw at or above it (the carry form needs t >= 1); a boundary equal to n
    // has none (its threshold would be 2^64)
    const uint32_t trips = threadIdx.x < n32 ? (n32 - threadIdx.x + BOOT_THREADS - 1) / BOOT_THREADS : 0u;
#pragma unroll
    for (int v = 0; v < 8; v++) {
        if (cum[v] == 0) ge[v] = trips;
        if (cum[v] >= n) ge[v] = 0;
    }
    // values 1..7 of this thread: ge[v-1] - ge[v]; warp sums go to the shared histogram
#pragma unroll
    for (int v = 1; v <= 7; v++) {
        uint32_t c = ge[v - 1] - ge[v];
        if (v >= 4 && !more_than_3) c = 0;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(&Hb[v], c);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t nz = 0;
        for (int v = 1; v <= 16; v++) nz += Hb[v];
        RatioOut r = ratio_lambda_hist(Hb, nz, P.min_count_correct);
        double ani = 0.;
        bool ok = r.ok && ani_from_lambda_dev(r.lambda, (double)P.k, nz, n, &ani);
        ok = ok && !isnan(ani) && !isnan(r.lambda);
        const uint64_t o = (uint64_t)row * BOOT_ITERS + it;
        res_ani[o] = ani;
        res_lambda[o] = r.lambda;
        res_ok[o] = ok ? 1 : 0;
    }
}

// Persistent kernel: the number of bootstrapped rows is read from device memory (no host round trip
// between the statistics kernel and the bootstrap).  One CTA per resident slot; the (row, iteration)
// items are handed out through a device counter, because their cost follows |genome_kmers| of the
// row and a fixed stride leaves the CTAs that drew the large rows running alone at the end.
__global__ void __launch_bounds__(BOOT_THREADS)  // forcing 6 CTAs/SM (40 registers) measured 9 % slower
k_boot_iter_p(const uint32_t *__restrict__ hist_in, const unsigned long long *__restrict__ d_nboot, uint64_t boot_cap, StatParams P,
              double *__restrict__ res_ani, double *__restrict__ res_lambda, uint8_t *__restrict__ res_ok,
              uint32_t *__restrict__ reject_flag, uint32_t *__restrict__ work_ctr) {
    __shared__ uint32_t Hb[17];
    __shared__ uint64_t cum[17];
    __shared__ uint64_t thr[16], nthr[16];
    __shared__ uint32_t s_item;
    const uint64_t nb = *d_nboot < boot_cap ? *d_nboot : boot_cap;
    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(work_ctr, 1u);
        __syncthreads();
        const uint64_t item = s_item;
        if (item >= nb * BOOT_ITERS) break;
        boot_one((uint32_t)(item / BOOT_ITERS), (uint32_t)(item % BOOT_ITERS), hist_in, P, res_ani, res_lambda, res_ok, reject_flag, Hb, cum, thr, nthr);
        __syncthreads();  // Hb / cum / s_item are rewritten by the next item
    }
}

// Exact sequential replay for a row whose counter-based draws hit Lemire's rejection branch
// (the redraw shifts the RNG stream). One thread per flagged row; practically never runs.
__global__ void k_boot_seq(const uint32_t *__restrict__ hist_in, uint32_t n_boot,
                           StatParams P, const uint32_t *__restrict__ reject_flag, double *__restrict__ res_ani,
                           double *__restrict__ res_lambda, uint8_t *__restrict__ res_ok,
                           const unsigned long long *__restrict__ d_nboot = nullptr) {
    const uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if (d_nboot && (unsigned long long)n_boot > *d_nboot) n_boot = (uint32_t)*d_nboot;  // n_boot = capacity then
    if (row >= n_boot || !reject_flag[row]) return;
    const uint32_t *H = hist_in + (uint64_t)row * 17;
    uint64_t cum[17], acc = 0;
    for (int v = 0; v < 17; v++) { acc += H[v]; cum[v] = acc; }
    const uint64_t n = acc;
    uint64_t state = 7ull;
    for (int it = 0; it < BOOT_ITERS; it++) {
        uint32_t Hb[17];
        for (int v = 0; v < 17; v++) Hb[v] = 0;
        for (uint64_t j = 0; j < n; j++) {
            uint64_t hi, lo;
            for (;;) {
                state += 0x2d358dccaa6c78a5ull;
                const uint64_t tt = state ^ 0x8bb84b93962eacc9ull;
                const uint64_t x = (state * tt) ^ __umul64hi(state, tt);
                hi = __umul64hi(x, n);
                lo = x * n;
                if (lo < n) {
                    const uint64_t t = (0ull - n) % n;
                    if (lo < t) continue;
                }
                break;
            }
            uint32_t v = 0;
            for (int q = 0; q < 16; q++) v += (hi >= cum[q]) ? 1u : 0u;
            Hb[v]++;
        }
        uint32_t nz = 0;
        for (int v = 1; v <= 16; v++) nz += Hb[v];
        RatioOut r = ratio_lambda_hist(Hb, nz, P.min_count_correct);
        double ani = 0.;
        bool ok = r.ok && ani_from_lambda_dev(r.lambda, (double)P.k, nz, n, &ani);
        ok = ok && !isnan(ani) && !isnan(r.lambda);
        const uint64_t o = (uint64_t)row * BOOT_ITERS + it;
        res_ani[o] = ani;
        res_lambda[o] = r.lambda;
        res_ok[o] = ok ? 1 : 0;
    }
}

// percentile pick (:885-896): of the successful iterations take the elements of rank suc*5/100-1
// and suc*95/100-1 of each list (sorted independently).  One 128-thread block per row; ranks by
// counting, so no sort is needed.
__global__ void __launch_bounds__(128)
k_boot_final(const uint32_t *__restrict__ boot_rows, uint32_t n_boot, const double *__restrict__ res_ani,
             const double *__restrict__ res_lambda, const uint8_t *__restrict__ res_ok,
             syl_ani_row *__restrict__ rows, const unsigned long long *__restrict__ d_nboot = nullptr) {
    __shared__ double a[BOOT_ITERS], l[BOOT_ITERS];
    __shared__ int s_suc;
    const uint32_t row = blockIdx.x;
    if (d_nboot && (unsigned long long)n_boot > *d_nboot) n_boot = (uint32_t)*d_nboot;  // n_boot = capacity then
    if (row >= n_boot) return;
    const int t = threadIdx.x;
    if (t == 0) {  // compact the successful iterations (order is irrelevant for rank selection)
        int suc = 0;
        for (int it = 0; it < BOOT_ITERS; it++) {
            const uint64_t o = (uint64_t)row * BOOT_ITERS + it;
            if (res_ok[o]) { a[suc] = res_ani[o]; l[suc] = res_lambda[o]; suc++; }
        }
        s_suc = suc;
    }
    __syncthreads();
    const int suc = s_suc;
    syl_ani_row &r = rows[boot_rows[row]];
    if (suc < 50) { if (t == 0) r.ci_valid = 0; return; }
    const int lo = suc * 5 / 100 - 1, hi = suc * 95 / 100 - 1;
    if (t < suc) {
        int ra = 0, rl = 0;
        const double x = a[t], y = l[t];
        for (int j = 0; j < suc; j++) {
            ra += (a[j] < x) || (a[j] == x && j < t);
            rl += (l[j] < y) || (l[j] == y && j < t);
        }
        if (ra == lo) r.ci[0] = x;
        if (ra == hi) r.ci[1] = x;
        if (rl == lo) r.ci[2] = y;
        if (rl == hi) r.ci[3] = y;
    }
    if (t == 0) r.ci_valid = 1;
}

static StatParams make_params(const syl_contain_params *p) {
    StatParams P;
    P.k = p->k;
    P.no_ci = p->no_ci;
    P.no_adj = p->no_adj;
    P.mean_coverage = p->mean_coverage;
    P.min_number_kmers = p->min_number_kmers;
    P.min_count_correct = p->min_count_correct;
    P.min_ani = p->minimum_ani >= 0. ? p->minimum_ani / 100. : (p->pseudotax ? 0.95 : 0.90);  // :746-748
    return P;
}

// ------------------------------------------------------------------------------------------------
// Staged query / profile: both get_stats passes, the winner decision and the bootstrap are enqueued
// back to back; the host synchronises ONCE, when it reads the final rows.
//   pass 1      k_join_hist + k_stats_hist -> rows appended to a per-rank ROW TABLE
//               (header {n_rows, n_boot, overflow} + R rows of 144 bytes, R fixed per call)
//   [N ranks: the caller all-gathers the row tables — collective 1]
//   ranking     k_rank_rows: every pass-1 survivor gets its position in the per-sample order
//               (final_est_ani descending, genome index ascending) — the reference's winner_table
//               (src/contain.rs:410-430) keeps, for every k-mer, the genome that comes first in that
//               order; ties go to the lowest genome index (its own tie winner is timing dependent)
//   winner      k_local_best: per sample key, the smallest order among the genomes (kept or tracked
//               k-mers) of its equal range in THIS shard
//   [N ranks: the caller all-reduces (MIN) the winner array — collective 2]
//   pass 2      k_join2_order (hit counts / lost k-mers against the winner) + k_stats_hist + bootstrap
//   [N ranks: the caller all-gathers the pass-2 row tables — collective 3]
//   finish      D2H of the table(s), derep_if_reassign_threshold (:353-375), abundances (:319-326), sort
// Single GPU: the winner minimum is taken inside k_join2_order and nothing is gathered.  A coverage
// count >= COV_BINS or more rows than the table holds is reported in the header; the caller then
// redoes the call in the CSR formulation or with a larger table.
// CSR formulation: k_join_hist<probe only> records the equal ranges and k_join2_order<.., CSR_*> walks
// them twice per pass (count hits per pair, CUB scan, scatter the hits' sample counts), with no winner in
// pass 1; k_stats replaces k_stats_hist; ranking, bootstrap and finish are shared.  Sizing the value
// array after the pass-1 scan costs a second host synchronisation, inside stage 1 (before any collective);
// pass 2 needs none, because its hits are a subset of pass 1's (same ranges, winners only).  Both
// formulations write the same row tables, so the ranks of a sharded profile may each run either one.
constexpr uint32_t ORD_NONE = 0x7F7F7F7Fu;  // memset-able; valid as int32 for the MIN all-reduce

struct ShardTable { unsigned long long n_rows, n_boot, ovf, pad; };
static_assert(sizeof(ShardTable) == 32, "table header");
static inline size_t table_bytes(uint64_t R) { return sizeof(ShardTable) + R * sizeof(syl_ani_row); }
__host__ __device__ static inline syl_ani_row *table_rows(void *t) { return reinterpret_cast<syl_ani_row *>(reinterpret_cast<uint8_t *>(t) + sizeof(ShardTable)); }

// order of every pass-1 row inside its sample; rows of this rank also land in the dense order table.
// `tabs`: `world` tables of `tbytes` bytes each (R rows capacity, R a multiple of 256)
__global__ void __launch_bounds__(256)
k_rank_rows(const uint8_t *__restrict__ tabs, uint64_t tbytes, uint32_t world, uint32_t R, uint32_t rank, uint64_t G,
            uint32_t genome_base, uint32_t *__restrict__ order_tbl) {
    __shared__ uint32_t s_smp[256], s_gen[256];
    __shared__ double s_ani[256];
    const uint64_t total = (uint64_t)world * R;
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    bool valid = false;
    uint32_t ms = 0, mg = 0, mr = 0;
    double ma = 0.;
    if (i < total) {
        mr = (uint32_t)(i / R);
        const uint32_t idx = (uint32_t)(i % R);
        const ShardTable *t = reinterpret_cast<const ShardTable *>(tabs + (uint64_t)mr * tbytes);
        if (idx < t->n_rows) {
            const syl_ani_row *row = reinterpret_cast<const syl_ani_row *>(reinterpret_cast<const uint8_t *>(t) + sizeof(ShardTable)) + idx;
            valid = true; ms = row->sample; mg = row->genome; ma = row->final_est_ani;
        }
    }
    uint32_t ord = 0;
    for (uint32_t r = 0; r < world; r++) {
        const ShardTable *t = reinterpret_cast<const ShardTable *>(tabs + (uint64_t)r * tbytes);
        const uint32_t n = t->n_rows < R ? (uint32_t)t->n_rows : R;
        const syl_ani_row *rows = reinterpret_cast<const syl_ani_row *>(reinterpret_cast<const uint8_t *>(t) + sizeof(ShardTable));
        for (uint32_t base = 0; base < n; base += 256) {  // uniform trip count
            const uint32_t j = base + threadIdx.x;
            if (j < n) { s_smp[threadIdx.x] = rows[j].sample; s_gen[threadIdx.x] = rows[j].genome; s_ani[threadIdx.x] = rows[j].final_est_ani; }
            else s_smp[threadIdx.x] = 0xFFFFFFFFu;
            __syncthreads();
            if (valid) {
                const uint32_t m = min(256u, n - base);
                for (uint32_t q = 0; q < m; q++)
                    ord += (s_smp[q] == ms && (s_ani[q] > ma || (s_ani[q] == ma && s_gen[q] < mg))) ? 1u : 0u;
            }
            __syncthreads();
        }
    }
    if (valid && mr == rank) order_tbl[(uint64_t)ms * G + (mg - genome_base)] = ord;
}

// smallest order (in the sample's row `ord` of the order table) among the genomes of the equal range [lo, e); kept
// and tracked k-mers both count (src/contain.rs:416-426)
__device__ __forceinline__ uint32_t range_winner(const uint32_t *__restrict__ gid, const uint32_t *__restrict__ ord, uint32_t lo,
                                                 uint32_t e) {
    uint32_t winner = ORD_NONE;
    walk_range<true>(gid, lo, e, [&](const uint32_t g) { winner = min(winner, ord[g]); });
    return winner;
}

// per sample key: the winner of its equal range in this shard
__global__ void k_local_best(const SampleView *__restrict__ views, uint64_t G, const uint32_t *__restrict__ gid,
                             const uint2 *__restrict__ hits, uint64_t hits_stride, const uint32_t *__restrict__ order_tbl,
                             uint32_t *__restrict__ wbest, const KeyMap km) {
  for_each_key(km, views, [&](const uint32_t smp, const uint64_t i) {
    const uint2 h = hits[(uint64_t)smp * hits_stride + i];
    wbest[(uint64_t)smp * hits_stride + i] = range_winner(gid, order_tbl + (uint64_t)smp * G, h.x, h.x + h.y);
  });
}

// Which hits of a walk count.  WIN_NONE (pass 1): every kept hit.  Pass 2: only the winner's, and every other pass-1
// survivor of the range loses the k-mer; the winner is the range's smallest order (WIN_FUSED, single GPU) or comes
// from wbest, all-reduced over the shards (WIN_GIVEN).
enum Winner { WIN_NONE, WIN_FUSED, WIN_GIVEN };

// a walk over the equal ranges recorded by k_join_hist
template <Winner W, JoinOut OUT>
__global__ void k_join2_order(const SampleView *__restrict__ views, uint64_t G, const uint32_t *__restrict__ gid,
                              const uint2 *__restrict__ hits, uint64_t hits_stride, const uint32_t *__restrict__ order_tbl,
                              const uint32_t *__restrict__ wbest, uint32_t *__restrict__ lost, const PairOut out, const KeyMap km) {
  for_each_key(km, views, [&](const uint32_t smp, const uint64_t i) {
    const uint2 h = hits[(uint64_t)smp * hits_stride + i];
    if (h.y == 0) return;
    const uint64_t row = (uint64_t)smp * G;
    const uint32_t *ord = W == WIN_NONE ? nullptr : order_tbl + row;
    const uint32_t lo = h.x, e = h.x + h.y, c = views[smp].count[i];
    uint32_t winner = ORD_NONE;
    if (W == WIN_FUSED) winner = range_winner(gid, ord, lo, e);
    if (W == WIN_GIVEN) winner = wbest[(uint64_t)smp * hits_stride + i];
    if (W != WIN_NONE && winner == ORD_NONE) return;  // no survivor holds this k-mer
    walk_range(gid, lo, e, [&](const uint32_t g) {
        if (W != WIN_NONE) {
            const uint32_t o = ord[g];
            if (o == ORD_NONE) return;                 // not a pass-1 survivor
            if (o != winner) {                         // src/contain.rs:641-646
                if (OUT != JOIN_CSR_FILL) atomicAdd(&lost[row + g], 1u);
                return;
            }
        }
        out.hit<OUT>(row + g, c);
    });
  });
}

// SYL_OK when `bytes` more keep the ctx within room->limit (its cached free blocks are handed back first if they are
// what stands in the way; that waits for the ctx stream), else SPLIT_BATCH
static int take_room(syl_ctx *ctx, JoinRoom *room, uint64_t bytes) {
    if (!room || !room->limit) return SYL_OK;
    auto held = [ctx] { return (uint64_t)(ctx->cached_bytes + ctx->transient_bytes); };
    if (held() + bytes > room->limit && !ctx->free_blocks.empty()) SYL_TRY(cache_trim(ctx));
    if (held() + bytes <= room->limit) return SYL_OK;
    room->want = bytes;
    return SPLIT_BATCH;
}

}  // namespace syl

// One in-flight device-driven query / profile (C ABI: syl_profile_job).
struct syl_profile_job {
    syl_ctx *ctx = nullptr;
    const syl_db *db = nullptr;
    syl::StatParams P;       // pass-2 / query parameters
    bool profile = true;
    double redundant_ani = 99.;
    double read_seq_id = -1.;            // > 0: -u with an explicit read identity
    std::vector<syl::SampleMeta> metas;  // per sample (only filled for -u)
    uint32_t S = 0, world = 1, rank = 0;
    uint64_t G = 0, R = 0, max_n = 0, tbytes = 0;
    int stage = 0;           // 1 pass 1 enqueued, 2 ranked, 3 pass 2 enqueued
    bool csr = false;        // CSR formulation instead of the per-pair count histograms
    syl::JoinRoom *room = nullptr;  // bound on the CSR hit values (host-sample batches only)
    syl::DevBuf<syl::SampleView> views;
    syl::DevBuf<uint8_t> touched, tab1, gat1, tab2, gat2, res_ok, scan_tmp;
    syl::DevBuf<uint32_t> chist, lost, order, contain1, wbest, boot_rows, hist, reject, range_bounds;
    syl::DevBuf<uint32_t> cnt, cursor, covs;   // CSR formulation
    syl::DevBuf<uint64_t> off;
    size_t scan_bytes = 0;
    syl::KeyMap km{nullptr, 0, 0};   // tiled (range, sample) mapping of the join kernels when there are several samples
    dim3 jgrid;
    syl::DevBuf<uint2> hits;
    syl::DevBuf<double> res_ani, res_lambda;
    syl::DevBuf<uint64_t> gn_size;
    std::vector<uint8_t> h_tab;
    syl::ScanChunk scan{};   // scan.kmers != nullptr: pass 1 by the scan formulation
};

namespace syl {
// estimate_true_cov (src/contain.rs:377-389) for the rows of one call (query: all rows; profile: the kept rows)
static inline double unknown_multiplier(const SampleMeta &m, int k) { return m.mean_read_length / (m.mean_read_length - (double)k + 1.); }

// Row-table capacity when the caller gives none, a multiple of 256.  The ranks of a sharded profile gather their tables
// with fixed-size collectives, so at world > 1 it depends on the sample count only (shards of 257 and 256 genomes
// would otherwise get 512 and 256 rows); one GPU also caps it at the number of pairs.
static uint64_t default_rows_per_rank(uint32_t S, uint64_t G, uint32_t world) {
    uint64_t R = 256 + 96ull * S;
    if (world == 1) R = std::min<uint64_t>((uint64_t)S * G, R);
    return (std::max<uint64_t>(R, 256) + 255) & ~255ull;
}

static bool histograms_fit(uint64_t n_pairs) { return n_pairs * COV_BINS * 4 <= (8ull << 30); }

// the per-pair outputs of pass 1 or 2 (the overflow counter is in that pass's row table)
static PairOut pair_out(const syl_profile_job *j, bool pass2) {
    ShardTable *t = reinterpret_cast<ShardTable *>(pass2 ? j->tab2.p : j->tab1.p);
    return PairOut{j->touched.p, j->chist.p, &t->ovf, j->cnt.p, j->off.p, j->cursor.p, j->covs.p};
}

// zeroes the per-pair buffers that a pass adds into
static int clear_pairs(syl_profile_job *j) {
    cudaStream_t st = j->ctx->stream;
    const uint64_t NP = (uint64_t)j->S * j->G;
    if (j->csr) {
        SYL_CUDA(cudaMemsetAsync(j->cnt.p, 0, (NP + 1) * 4, st));  // cnt[NP] = 0: off[NP] is the total
        SYL_CUDA(cudaMemsetAsync(j->cursor.p, 0, NP * 4, st));
    } else {
        SYL_CUDA(cudaMemsetAsync(j->touched.p, 0, NP, st));
        SYL_CUDA(cudaMemsetAsync(j->chist.p, 0, NP * COV_BINS * 4, st));
    }
    return SYL_OK;
}

// One walk over the equal ranges in j->hits into OUT.  Pass 1 walks only in the CSR formulation (the histogram one
// accumulates inside the probe) and counts every kept hit.  Pass 2 counts the winner's hits, with the winner taken in
// the walk on one GPU and from the all-reduced wbest across ranks.
template <JoinOut OUT>
static void join_walk(syl_profile_job *j, bool pass2) {
    const syl_db *db = j->db;
    if (j->scan.kmers) {
        if (!j->max_n || !j->scan.n) return;
        KernelTimer kt(j->ctx, SYL_KERNEL_SCAN);
        k_scan<OUT><<<nblk(j->scan.n, (uint64_t)SCAN_THREADS * SCAN_PER_THREAD), SCAN_THREADS, 0, j->ctx->stream>>>(j->scan, j->S, j->G,
                                                                                                            pair_out(j, pass2));
        j->ctx->launches++;
        return;
    }
    if (!j->max_n || !db->N) return;
    auto k = j->world > 1 ? k_join2_order<WIN_GIVEN, OUT> : k_join2_order<WIN_FUSED, OUT>;
    if constexpr (OUT != JOIN_HIST) {
        if (!pass2) k = k_join2_order<WIN_NONE, OUT>;
    }
    KernelTimer kt(j->ctx, pass2 ? SYL_KERNEL_JOIN2 : SYL_KERNEL_JOIN);
    k<<<j->jgrid, 128, 0, j->ctx->stream>>>(j->views.p, j->G, db->gid, j->hits.p, j->max_n, j->order.p, j->wbest.p, j->lost.p,
                                            pair_out(j, pass2), j->km);
    j->ctx->launches++;
}

// CSR formulation of one pass over the equal ranges in j->hits: count walk, scan, fill walk.  Pass 1 sizes covs,
// which needs a host synchronisation; pass 2's hits are a subset of pass 1's, so that size bounds them as well.
static int csr_walks(syl_profile_job *j, bool pass2) {
    syl_ctx *ctx = j->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t NP = (uint64_t)j->S * j->G;
    join_walk<JOIN_CSR_COUNT>(j, pass2);
    size_t tb = j->scan_bytes;
    SYL_CUDA(cub::DeviceScan::ExclusiveSum(j->scan_tmp.p, tb, j->cnt.p, j->off.p, (int)(NP + 1), st));
    if (!pass2) {
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_COVS_TOTAL, j->off.p + NP, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        const uint64_t total = std::max<uint64_t>(ctx->h_counters[CNT_COVS_TOTAL], 1);
        SYL_TRY(take_room(ctx, j->room, (total * 4 + 255) & ~255ull));
        SYL_TRY(j->covs.alloc(total, st));
    }
    join_walk<JOIN_CSR_FILL>(j, pass2);
    SYL_CUDA(cudaGetLastError());
    return SYL_OK;
}

// statistics of one pass (either formulation) into the row table `tab`
static int enqueue_stats(syl_profile_job *j, const StatParams &P, bool pass2, void *tab, const StatExtra &X) {
    syl_ctx *ctx = j->ctx;
    const syl_db *db = j->db;
    const uint64_t NP = (uint64_t)j->S * j->G;
    ShardTable *t = reinterpret_cast<ShardTable *>(tab);
    uint32_t *lost = pass2 ? j->lost.p : nullptr;
    if (NP == 0) return SYL_OK;  // an empty shard: no pairs, the table keeps its zeroed header
    KernelTimer kt(ctx, SYL_KERNEL_STATS);
    if (j->csr)
        k_stats<<<nblk(NP, STAT_WARPS), STAT_WARPS * 32, 0, ctx->stream>>>(j->cnt.p, j->off.p, j->covs.p, db->glen, lost, j->G, NP, db->genome_base,
                                                                          P, pass2 ? 1 : 0, table_rows(tab), j->R, j->boot_rows.p, j->hist.p, j->R,
                                                                          &t->n_rows, &t->n_boot, X);
    else
        k_stats_hist<<<nblk(NP, STAT_WARPS), STAT_WARPS * 32, 0, ctx->stream>>>(j->touched.p, j->chist.p, db->glen, lost, j->G, NP, db->genome_base,
                                                                               P, pass2 ? 1 : 0, table_rows(tab), j->R, j->boot_rows.p, j->hist.p, j->R,
                                                                               &t->n_rows, &t->n_boot, X);
    ctx->launches++;
    SYL_CUDA(cudaGetLastError());
    return SYL_OK;
}

// stage 1: allocate, pass 1 (P1 = the pass-1 parameters: profile skips the bootstrap there).  The one place that picks
// the formulation: CSR when the caller asks for it (a histogram run met a count >= COV_BINS), when SYL_CONTAIN_CSR is
// set (read per call) or when this job's per-pair histograms would exceed 8 GB.  The choice is local to the job: the
// ranks of a sharded profile may pick differently.
static int job_begin(syl_ctx *ctx, const syl_db *db, const SampleView *views, const SampleMeta *metas, uint32_t n_samples,
                     const syl_contain_params *p, bool profile, bool csr, uint32_t world, uint32_t rank, uint64_t R,
                     syl_profile_job **out, JoinRoom *room = nullptr, const ScanChunk *scan = nullptr) {
    cudaStream_t st = ctx->stream;
    Handle<syl_profile_job> h(new (std::nothrow) syl_profile_job());
    if (!h) return SYL_ERR_OOM;
    // the scan formulation is pass 1 of a query: pass 2 walks the winners of recorded index ranges, which a scan has not
    if (scan && profile) { set_error("the scan formulation runs query calls only"); return SYL_ERR_ARG; }
    syl_profile_job *j = h.get();
    const uint64_t NP = (uint64_t)n_samples * db->n_genomes;
    csr = csr || getenv("SYL_CONTAIN_CSR") != nullptr || !histograms_fit(NP);
    j->ctx = ctx; j->db = db; j->profile = profile; j->csr = csr; j->S = n_samples; j->G = db->n_genomes; j->world = world; j->rank = rank;
    j->room = room;
    if (scan) j->scan = *scan;
    syl_contain_params pp = *p;
    pp.pseudotax = profile ? 1 : 0;
    j->P = make_params(&pp);
    j->redundant_ani = pp.redundant_ani;
    if (p->estimate_unknown) { j->read_seq_id = p->read_seq_id; j->metas.assign(metas, metas + n_samples); }
    j->R = R ? ((R + 255) & ~255ull) : default_rows_per_rank(n_samples, db->n_genomes, world);
    j->tbytes = table_bytes(j->R);
    if (j->R * BOOT_ITERS >= 0xFFFF0000ull) { set_error("row capacity too large for the bootstrap work counter"); return SYL_ERR_ARG; }
    if (NP >= 0x7FFFFFFFull) { set_error("samples x genomes exceeds 2^31 pairs per call; split the sample batch"); return SYL_ERR_ARG; }
    std::vector<SampleView> hv(views, views + n_samples);
    for (const SampleView &v : hv) j->max_n = std::max<uint64_t>(j->max_n, v.n);
    const uint64_t HN = scan ? 1 : std::max<uint64_t>((uint64_t)j->S * j->max_n, 1);  // the scan records no ranges
    SYL_TRY(j->views.alloc(n_samples, st));
    if (csr) {
        SYL_TRY(j->cnt.alloc(NP + 1, st)); SYL_TRY(j->cursor.alloc(NP, st)); SYL_TRY(j->off.alloc(NP + 1, st));
        cub::DeviceScan::ExclusiveSum(nullptr, j->scan_bytes, j->cnt.p, j->off.p, (int)(NP + 1), st);
        SYL_TRY(j->scan_tmp.alloc(j->scan_bytes, st));
    } else {
        SYL_TRY(j->touched.alloc(NP, st)); SYL_TRY(j->chist.alloc(NP * COV_BINS, st));
    }
    SYL_TRY(j->hits.alloc(HN, st));
    SYL_TRY(j->tab1.alloc(j->tbytes, st));
    SYL_TRY(j->boot_rows.alloc(j->R, st)); SYL_TRY(j->hist.alloc(j->R * 17, st));
    SYL_TRY(j->res_ani.alloc(j->R * BOOT_ITERS, st)); SYL_TRY(j->res_lambda.alloc(j->R * BOOT_ITERS, st));
    SYL_TRY(j->res_ok.alloc(j->R * BOOT_ITERS, st)); SYL_TRY(j->reject.alloc(j->R + 1, st));  // [R] = the bootstrap's work counter
    if (profile) {
        SYL_TRY(j->lost.alloc(NP, st)); SYL_TRY(j->order.alloc(NP, st)); SYL_TRY(j->contain1.alloc(NP, st));
        SYL_TRY(j->tab2.alloc(j->tbytes, st)); SYL_TRY(j->gn_size.alloc(std::max<uint64_t>(j->G, 1), st));
        if (world > 1) { SYL_TRY(j->gat1.alloc(j->tbytes * world, st)); SYL_TRY(j->wbest.alloc(HN, st)); }
    }
    if (world > 1) SYL_TRY(j->gat2.alloc(j->tbytes * world, st));  // final tables of all ranks (profile: pass 2; query: pass 1)
    // a pageable source is staged by the driver before cudaMemcpyAsync returns: hv may go out of scope
    SYL_CUDA(cudaMemcpyAsync(j->views.p, hv.data(), n_samples * sizeof(SampleView), cudaMemcpyHostToDevice, st));
    if (profile && j->G) SYL_CUDA(cudaMemcpyAsync(j->gn_size.p, db->h_gn_size.data(), j->G * 8, cudaMemcpyHostToDevice, st));
    SYL_TRY(clear_pairs(j));
    SYL_CUDA(cudaMemsetAsync(j->hits.p, 0, HN * sizeof(uint2), st));
    SYL_CUDA(cudaMemsetAsync(j->tab1.p, 0, sizeof(ShardTable), st));
    j->jgrid = dim3(nblk(std::max<uint64_t>(j->max_n, 1), 128), (unsigned)j->S);
    static const bool tile_env_off = getenv("SYL_JOIN_PLAIN") != nullptr;
    if (j->S > 1 && j->max_n && db->N && !tile_env_off && !scan) {
        // ~100 keys of the largest sample per (range, sample) block; ranges are equal numbers of db buckets
        const uint64_t R = std::min<uint64_t>(std::max<uint64_t>(j->max_n / 100, 1), std::max<uint64_t>(db->NB, 1));
        const uint64_t bpr = (db->NB + R - 1) / R;
        if (R * j->S < 0x7FFFFFFFull) {
            SYL_TRY(j->range_bounds.alloc((uint64_t)j->S * (R + 1), st));
            KernelTimer kt(ctx, SYL_KERNEL_JOIN);
            k_range_bounds<<<nblk((uint64_t)j->S * (R + 1), 256), 256, 0, st>>>(j->views.p, j->S, (uint32_t)R, bpr, db->M, db->NB, j->range_bounds.p);
            ctx->launches++;
            j->km = KeyMap{j->range_bounds.p, (uint32_t)R, j->S};
            j->jgrid = dim3((unsigned)(R * j->S), 1);
        }
    }
    if (scan && !csr) join_walk<JOIN_HIST>(j, false);
    if (j->max_n && db->N && !scan) {
        KernelTimer kt(ctx, SYL_KERNEL_JOIN);
        const auto probe = csr ? k_join_hist<true> : k_join_hist<false>;
        probe<<<j->jgrid, 128, 0, st>>>(j->views.p, j->G, db->keys, db->gid, db->N, db->bstart, db->M, db->NB, db->maxkey,
                                        pair_out(j, false), j->hits.p, j->max_n, j->km);
        ctx->launches++;
    }
    if (csr) SYL_TRY(csr_walks(j, false));
    StatParams P1 = j->P;
    if (profile) P1.no_ci = 1;  // pass-1 confidence intervals are never reported (pass-2 rows replace them)
    StatExtra X;
    X.pair_stride = j->G;
    if (profile) X.contain1_out = j->contain1.p;
    SYL_TRY(enqueue_stats(j, P1, false, j->tab1.p, X));
    j->stage = 1;
    *out = h.release();
    return SYL_OK;
}

// bootstrap of the rows listed in table `tab` (device-side count)
static int job_bootstrap(syl_profile_job *j, void *tab) {
    syl_ctx *ctx = j->ctx;
    cudaStream_t st = ctx->stream;
    if (j->P.no_ci) return SYL_OK;
    ShardTable *t = reinterpret_cast<ShardTable *>(tab);
    SYL_CUDA(cudaMemsetAsync(j->reject.p, 0, (size_t)(j->R + 1) * 4, st));
    // test hook (read per call): flag every row, so k_boot_seq replays all of them sequentially; the flags are
    // reject[0..R) only, reject[R] is k_boot_iter_p's work counter and stays zero
    if (getenv("SYL_BOOT_REPLAY") != nullptr) SYL_CUDA(cudaMemsetAsync(j->reject.p, 1, (size_t)j->R * 4, st));
    KernelTimer kt(ctx, SYL_KERNEL_BOOT);
    // resident CTAs per SM (a partially filled second wave would double the tail); initialised once, because contexts
    // on other threads of the process may get here at the same time
    static const int boot_ctas = []() {
        int n = 0;
        return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_boot_iter_p, BOOT_THREADS, 0) == cudaSuccess ? n : 4;
    }();
    k_boot_iter_p<<<ctx->num_sms * std::max(boot_ctas, 1), BOOT_THREADS, 0, st>>>(j->hist.p, &t->n_boot, j->R, j->P, j->res_ani.p, j->res_lambda.p, j->res_ok.p, j->reject.p, j->reject.p + j->R);
    k_boot_seq<<<nblk(j->R, 32), 32, 0, st>>>(j->hist.p, (uint32_t)j->R, j->P, j->reject.p, j->res_ani.p, j->res_lambda.p, j->res_ok.p, &t->n_boot);
    k_boot_final<<<(unsigned)j->R, 128, 0, st>>>(j->boot_rows.p, (uint32_t)j->R, j->res_ani.p, j->res_lambda.p, j->res_ok.p, table_rows(tab), &t->n_boot);
    kt.stop();
    ctx->launches += 3;
    SYL_CUDA(cudaGetLastError());
    return SYL_OK;
}

// stage 2 (profile): order of the survivors from the gathered pass-1 tables, local winner candidates
static int job_rank(syl_profile_job *j) {
    syl_ctx *ctx = j->ctx;
    cudaStream_t st = ctx->stream;
    const syl_db *db = j->db;
    const uint64_t NP = (uint64_t)j->S * j->G;
    SYL_CUDA(cudaMemsetAsync(j->order.p, 0x7F, NP * 4, st));
    const uint8_t *tabs = j->world > 1 ? j->gat1.p : j->tab1.p;
    k_rank_rows<<<nblk((uint64_t)j->world * j->R, 256), 256, 0, st>>>(tabs, j->tbytes, j->world, (uint32_t)j->R, j->rank, j->G, db->genome_base, j->order.p);
    ctx->launches++;
    if (j->world > 1) {
        KernelTimer kt(ctx, SYL_KERNEL_JOIN2);
        k_local_best<<<j->jgrid, 128, 0, st>>>(j->views.p, j->G, db->gid, j->hits.p, j->max_n, j->order.p, j->wbest.p, j->km);
        ctx->launches++;
    }
    SYL_CUDA(cudaGetLastError());
    j->stage = 2;
    return SYL_OK;
}

// stage 3 (profile): pass 2 against the (all-reduced) winners, statistics, bootstrap
static int job_pass2(syl_profile_job *j) {
    syl_ctx *ctx = j->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t NP = (uint64_t)j->S * j->G;
    SYL_CUDA(cudaMemsetAsync(j->lost.p, 0, NP * 4, st));
    SYL_CUDA(cudaMemsetAsync(j->tab2.p, 0, sizeof(ShardTable), st));
    SYL_TRY(clear_pairs(j));
    if (j->csr) SYL_TRY(csr_walks(j, true));
    else join_walk<JOIN_HIST>(j, true);
    StatExtra X;
    X.pair_stride = j->G;
    X.contain1_in = j->contain1.p;
    X.gn_size = j->gn_size.p;
    SYL_TRY(enqueue_stats(j, j->P, true, j->tab2.p, X));
    SYL_TRY(job_bootstrap(j, j->tab2.p));
    j->stage = 3;
    return SYL_OK;
}

// derep_if_reassign_threshold (src/contain.rs:353-375) + abundances (:319-326) + the output order (:329-334)
// for the pass-2 rows of all shards: row.reserved = pass-1 containment count, row.seq_abund = genome size
static void profile_finalize(std::vector<syl_ani_row> &r2, uint32_t n_samples, int k, double redundant_ani, std::vector<syl_ani_row> &all,
                             const std::vector<SampleMeta> *metas = nullptr, double read_seq_id = -1.) {
    std::sort(r2.begin(), r2.end(), [](const syl_ani_row &a, const syl_ani_row &b) {
        return a.sample != b.sample ? a.sample < b.sample : a.genome < b.genome;
    });
    const double threshold = std::pow(redundant_ani / 100., (double)k);
    size_t i2 = 0;
    for (uint32_t smp = 0; smp < n_samples; smp++) {
        std::vector<syl_ani_row> kept;
        for (; i2 < r2.size() && r2[i2].sample == smp; i2++) {
            const syl_ani_row &n2 = r2[i2];
            const double num_reassign = (double)((uint64_t)n2.reserved - n2.contain);
            const double reass_thresh = threshold * (double)n2.glen;
            if (num_reassign < reass_thresh) kept.push_back(n2);
        }
        double bases_explained = 1.;
        if (metas && read_seq_id > 0.) {  // -u: estimate_true_cov (:310) + estimate_covered_bases (:391-408)
            const SampleMeta &m = (*metas)[smp];
            const double mult = unknown_multiplier(m, k), kid = std::pow(read_seq_id / 100., (double)k);
            double covered = 0.;
            for (syl_ani_row &r : kept) {
                r.final_est_cov = r.final_est_cov / kid * mult;
                covered += r.seq_abund * r.final_est_cov;  // seq_abund still holds gn_size
            }
            const double tentative = (double)(m.c * m.sum_counts) * mult;
            bases_explained = tentative == 0. ? 0. : std::min(covered / tentative, 1.);
        }
        double total_cov = 0., total_seq_cov = 0.;
        for (const syl_ani_row &r : kept) {
            total_cov += r.final_est_cov;
            total_seq_cov += r.final_est_cov * r.seq_abund;  // seq_abund still holds gn_size
        }
        for (syl_ani_row &r : kept) {
            const double gs = r.seq_abund;
            r.rel_abund = r.final_est_cov / total_cov * 100.;
            r.seq_abund = r.final_est_cov * gs / total_seq_cov * 100. * bases_explained;
            r.reserved = 0.;
        }
        std::stable_sort(kept.begin(), kept.end(),
                         [](const syl_ani_row &a, const syl_ani_row &b) { return a.rel_abund > b.rel_abund; });
        all.insert(all.end(), kept.begin(), kept.end());
    }
}

// last stage: read the final table(s); SYL_ERR_CAPACITY: *need_R rows per rank are needed;
// SYL_ERR_UNSUPPORTED: a coverage count >= COV_BINS somewhere (the call needs the CSR formulation)
static int job_finish(syl_profile_job *j, std::vector<syl_ani_row> &out, uint64_t *need_R) {
    syl_ctx *ctx = j->ctx;
    cudaStream_t st = ctx->stream;
    *need_R = 0;
    const uint32_t nt = j->world > 1 ? j->world : 1;
    const uint8_t *src = j->world > 1 ? j->gat2.p : (j->profile ? j->tab2.p : j->tab1.p);
    const uint8_t *src1 = (j->world > 1 && j->profile) ? j->gat1.p : j->tab1.p;  // pass-1 tables: only their headers matter here
    const size_t bytes = j->tbytes * nt;
    j->h_tab.resize(bytes + sizeof(ShardTable) * nt);
    SYL_CUDA(cudaMemcpyAsync(j->h_tab.data(), src, bytes, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpy2DAsync(j->h_tab.data() + bytes, sizeof(ShardTable), src1, j->tbytes, sizeof(ShardTable),
                               (j->world > 1 && j->profile) ? nt : 1, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));  // the one synchronisation of the call
    bool ovf = false;
    uint64_t need = 0;
    std::vector<syl_ani_row> rows;
    for (uint32_t r = 0; r < ((j->world > 1 && j->profile) ? nt : 1); r++) {  // every rank reaches the same verdict
        const ShardTable *h1 = reinterpret_cast<const ShardTable *>(j->h_tab.data() + bytes) + r;
        ovf |= h1->ovf != 0;
        need = std::max<uint64_t>(need, h1->n_rows);
    }
    for (uint32_t r = 0; r < nt; r++) {
        const ShardTable *t = reinterpret_cast<const ShardTable *>(j->h_tab.data() + (size_t)r * j->tbytes);
        ovf |= t->ovf != 0;
        need = std::max<uint64_t>(need, std::max(t->n_rows, t->n_boot));
        const syl_ani_row *tr = reinterpret_cast<const syl_ani_row *>(reinterpret_cast<const uint8_t *>(t) + sizeof(ShardTable));
        for (uint64_t i = 0; i < std::min<uint64_t>(t->n_rows, j->R); i++) rows.push_back(tr[i]);
    }
    if (ovf) { set_error("coverage count >= 256: CSR formulation needed"); return SYL_ERR_UNSUPPORTED; }
    if (need > j->R) { *need_R = need; set_error("row table too small"); return SYL_ERR_CAPACITY; }
    if (j->profile) {
        profile_finalize(rows, j->S, j->P.k, j->redundant_ani, out, &j->metas, j->read_seq_id);
    } else {
        std::sort(rows.begin(), rows.end(), [](const syl_ani_row &a, const syl_ani_row &b) {
            return a.sample != b.sample ? a.sample < b.sample : a.genome < b.genome;
        });
        if (j->read_seq_id > 0.)  // estimate_true_cov (:295)
            for (syl_ani_row &r : rows) {
                const SampleMeta &m = j->metas[r.sample];
                r.final_est_cov = r.final_est_cov / std::pow(j->read_seq_id / 100., (double)j->P.k) * unknown_multiplier(m, j->P.k);
            }
        out.swap(rows);
    }
    return SYL_OK;
}

// single-GPU driver of the stages for syl_query / syl_profile.  A histogram run that met a count >= COV_BINS is redone
// in the CSR formulation (job_begin may also take it up front); a row table that is too small is redone with the size
// it needed.
// `overlap`, when given, runs once, after the first attempt's stages are enqueued and before its result is awaited (the
// host samples stage their next batch there).  `room` (host-sample batches) bounds what the joins allocate beyond the
// batch's plan: CSR hit values or a capacity retry's row tables that do not fit it rerun the samples as two halves on
// the same views, recursively, and a single sample that does not fit is SYL_ERR_OOM.
int contain_fast(syl_ctx *ctx, const syl_db *db, const SampleView *views, const SampleMeta *metas, uint32_t n_samples,
                 const syl_contain_params *p, bool profile, std::vector<syl_ani_row> &out, const std::function<int()> &overlap,
                 JoinRoom *room, const ScanChunk *scan) {
    uint64_t R = 0;
    bool csr = false;
    bool overlapped = false;
    for (int attempt = 0; attempt < 4; attempt++) {  // one formulation switch + capacity retries
        syl_profile_job *j = nullptr;
        int rc = job_begin(ctx, db, views, metas, n_samples, p, profile, csr, 1, 0, R, &j, room, scan);
        if (rc == SYL_OK) {
            if (profile) {
                rc = job_rank(j);
                if (rc == SYL_OK) rc = job_pass2(j);
            } else {
                rc = job_bootstrap(j, j->tab1.p);
            }
            if (rc == SYL_OK && !overlapped && overlap) { overlapped = true; rc = overlap(); }
            uint64_t need = 0;
            if (rc == SYL_OK) rc = job_finish(j, out, &need);
            if (rc == SYL_ERR_CAPACITY) {
                R = need + 256;
                // the retry reuses this job's blocks and adds row tables for R rows (a few KB for rounding)
                const int room_rc = take_room(ctx, room, ((R + 255) & ~255ull) * ROW_BYTES + 4096);
                if (room_rc != SYL_OK) rc = room_rc;
            }
            syl_profile_job_free(j);
        }
        if (rc == SYL_ERR_CAPACITY) { out.clear(); continue; }
        if (rc == SYL_ERR_UNSUPPORTED && !csr) { csr = true; out.clear(); continue; }  // a count >= COV_BINS
        if (rc != SPLIT_BATCH) return rc;
        out.clear();
        if (n_samples == 1) {
            set_error("sample " + std::to_string(room->s0) + " needs " + std::to_string(room->want) +
                      " more bytes of device memory for its joins, the budget is " + std::to_string(room->budget) + " bytes");
            return SYL_ERR_OOM;
        }
        SYL_TRY(cache_trim(ctx));  // the halves allocate to their own sizes, not next to this job's cached blocks
        const uint32_t h = n_samples / 2;
        if (debug_timing())
            fprintf(stderr, "[join split] samples %u..%u: %llu bytes do not fit, halves of %u and %u samples\n", room->s0,
                    room->s0 + n_samples, (unsigned long long)room->want, h, n_samples - h);
        JoinRoom r0 = *room, r1 = *room;
        r1.s0 += h;
        std::vector<syl_ani_row> second;
        ScanChunk s1{};
        if (scan) { s1 = *scan; s1.tables += h; }
        SYL_TRY(contain_fast(ctx, db, views, metas, h, p, profile, out, overlapped ? std::function<int()>() : overlap, &r0, scan));
        SYL_TRY(contain_fast(ctx, db, views + h, metas + h, n_samples - h, p, profile, second, {}, &r1, scan ? &s1 : nullptr));
        for (syl_ani_row &r : second) {
            r.sample += h;
            out.push_back(r);
        }
        return SYL_OK;
    }
    return SYL_ERR_CAPACITY;
}

}  // namespace syl

using namespace syl;

extern "C" {

void syl_contain_params_default(syl_contain_params *p, int k, int pseudotax) {
    if (!p) return;
    p->k = k;
    p->pseudotax = pseudotax;
    p->no_ci = 0;
    p->no_adj = 0;
    p->mean_coverage = 0;
    p->estimate_unknown = 0;
    p->read_seq_id = -1.;
    p->min_number_kmers = 50.;
    p->min_count_correct = 3.;
    p->minimum_ani = -1.;
    p->redundant_ani = 99.;
}

int syl_profile_shard_begin(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                            const syl_contain_params *p, uint32_t world, uint32_t rank, uint64_t rows_per_rank, int csr,
                            syl_profile_job **out) {
    uint64_t dummy = 0;
    if (!out || !db) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    if (world == 0 || rank >= world || n_samples == 0) { set_error("bad world / rank / sample count"); return SYL_ERR_ARG; }
    SYL_TRY(check_contain_args(ctx, db->k, db->c, db->has_tracked, true, samples, n_samples, p, nullptr, 0, &dummy));
    SYL_ENTER(ctx);
    std::vector<SampleView> views;
    std::vector<SampleMeta> metas;
    SYL_TRY(handle_views(ctx, samples, n_samples, p->estimate_unknown != 0, views, metas));
    return job_begin(ctx, db, views.data(), metas.data(), n_samples, p, true, csr != 0, world, rank, rows_per_rank, out);
}

int syl_profile_job_buffers(const syl_profile_job *j, void **d_table1, void **d_gathered1, uint64_t *table_bytes,
                            void **d_winner, uint64_t *winner_elems, void **d_table2, void **d_gathered2) {
    if (!j) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (d_table1) *d_table1 = j->tab1.p;
    if (d_gathered1) *d_gathered1 = j->gat1.p;
    if (table_bytes) *table_bytes = j->tbytes;
    if (d_winner) *d_winner = j->wbest.p;
    if (winner_elems) *winner_elems = std::max<uint64_t>((uint64_t)j->S * j->max_n, 1);
    if (d_table2) *d_table2 = j->tab2.p;
    if (d_gathered2) *d_gathered2 = j->gat2.p;
    return SYL_OK;
}

int syl_profile_shard_rank(syl_profile_job *j) {
    if (!j || j->stage != 1 || !j->profile) { set_error("profile job: wrong stage"); return SYL_ERR_ARG; }
    SYL_ENTER(j->ctx);
    return job_rank(j);
}

int syl_profile_shard_pass2(syl_profile_job *j) {
    if (!j || j->stage != 2) { set_error("profile job: wrong stage"); return SYL_ERR_ARG; }
    SYL_ENTER(j->ctx);
    return job_pass2(j);
}

int syl_profile_shard_finish(syl_profile_job *j, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows, uint64_t *need_rows_per_rank) {
    if (!j || j->stage != 3 || !n_rows || (cap && !rows)) { set_error("profile job: wrong stage / NULL argument"); return SYL_ERR_ARG; }
    SYL_ENTER(j->ctx);
    std::vector<syl_ani_row> out;
    uint64_t need = 0;
    const int rc = job_finish(j, out, &need);
    if (need_rows_per_rank) *need_rows_per_rank = need;
    if (rc != SYL_OK) return rc;
    return copy_rows(out, rows, cap, n_rows);
}

void syl_profile_job_free(syl_profile_job *j) {
    delete j;  // the scratch blocks go back to the owning ctx's cache (DevBuf::owner)
}

}  // extern "C"
