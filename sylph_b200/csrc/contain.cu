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
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <new>
#include <vector>

#include "common.cuh"
#include "crmath.cuh"
#include "ingest.hpp"
#include "sample_batches.hpp"
#include "shard_cut.hpp"

struct syl_db {
    int device = 0;
    syl_ctx *owner = nullptr;       // arrays are blocks of this ctx's cache
    cudaStream_t stream = nullptr;
    uint64_t n_genomes = 0;
    uint32_t genome_base = 0;
    uint64_t N = 0;             // index entries (genome_kmers + tracked)
    uint64_t *keys = nullptr;   // sorted ascending
    uint32_t *gid = nullptr;    // (genome << 1) | is_tracked
    uint32_t *bstart = nullptr; // NB + 1 bucket starts
    uint64_t NB = 0, M = 0, maxkey = 0;
    uint32_t *glen = nullptr;   // |genome_kmers| per genome (device)
    std::vector<uint64_t> h_gn_size;
    int has_tracked = 0;
    int k = 31;
    uint64_t c = 200;
};

namespace syl {

static inline unsigned nblk(uint64_t n, int bs) { return (unsigned)((n + bs - 1) / bs); }

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

// ---- index build ----------------------------------------------------------------------------
//
// The index is every entry (key, gid = genome << 1 | tracked) of the db in (key, tracked, genome) order: the order of a
// stable sort of all genomes' k-mers in genome order followed by all tracked k-mers in genome order (entries equal in
// key and gid cannot be told apart).  It is built without a global sort: a max pass fixes the bucket directory
// (bucket_of below), a histogram pass counts each bucket, a scatter pass writes every entry into its bucket's segment
// of the final arrays, and each bucket is then sorted on its own.  Every pass reads the input as CSR chunks
// (DbChunk): a device source is one chunk, a host source is cut into chunks that are copied while the previous
// chunk's kernels run, so the build needs device memory for the index and two staging chunks, not for a sort.

__global__ void k_glen(const uint64_t *__restrict__ kmer_off, uint64_t n_genomes, uint32_t *__restrict__ glen) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < n_genomes) glen[g] = (uint32_t)(kmer_off[g + 1] - kmer_off[g]);
}

__device__ __forceinline__ uint64_t bucket_of(uint64_t key, uint64_t M, uint64_t NB) {
    uint64_t b = __umul64hi(key, M);
    return b < NB ? b : NB - 1;
}

// One chunk of the build's input: up to two segments, each a run of entries of one part (0 = genome k-mers,
// 1 = tracked k-mers).  Segment s holds keys[s][0 .. n[s]) of part part[s], its part-local entries p0[s] .. p0[s] + n[s];
// off[s] is the slice of that part's offsets of genomes g0[s] .. g0[s] + n_off[s] - 1 (values part-local, as given).
struct DbChunk {
    const uint64_t *keys[2];
    const uint64_t *off[2];
    uint64_t n_off[2], g0[2], p0[2], n[2];
    uint32_t part[2];
};

// (key, tracked, genome) order of an entry inside its key: the gid rotated so that the tracked bit leads (genome < 2^31 - 1)
__device__ __forceinline__ uint32_t gid_rank(uint32_t gid) { return (gid >> 1) | (gid << 31); }
__device__ __forceinline__ uint32_t rank_gid(uint32_t r) { return (r << 1) | (r >> 31); }
__device__ __forceinline__ bool entry_less(uint64_t ka, uint32_t ra, uint64_t kb, uint32_t rb) {
    return ka < kb || (ka == kb && ra < rb);
}

__device__ __forceinline__ uint64_t chunk_key(const DbChunk &c, uint64_t i) {
    return i < c.n[0] ? c.keys[0][i] : c.keys[1][i - c.n[0]];
}

__global__ void __launch_bounds__(256) k_db_max(DbChunk c, unsigned long long *__restrict__ mx) {
    uint64_t m = 0;
    const uint64_t n = c.n[0] + c.n[1];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        m = max(m, chunk_key(c, i));
    for (int o = 16; o; o >>= 1) m = max(m, (uint64_t)__shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(mx, (unsigned long long)m);
}

// bucket b is counted in slot[b + 2]: the inclusive scan of the slots then leaves bucket b's start in slot[b + 1],
// where k_db_scatter uses it as the bucket's cursor
__global__ void __launch_bounds__(256) k_db_hist(DbChunk c, uint64_t M, uint64_t NB, uint32_t *__restrict__ slot) {
    const uint64_t n = c.n[0] + c.n[1];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        atomicAdd(slot + bucket_of(chunk_key(c, i), M, NB) + 2, 1u);
}

// every entry to the next free place of its bucket; afterwards slot[b + 1] has advanced to the start of bucket b + 1,
// so slot[0 .. NB] is the bucket directory
__global__ void __launch_bounds__(256) k_db_scatter(DbChunk c, uint64_t M, uint64_t NB, uint32_t *__restrict__ slot,
                                                    uint64_t *__restrict__ keys, uint32_t *__restrict__ gid) {
    const uint64_t n = c.n[0] + c.n[1];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const bool s = i >= c.n[0];
        const uint64_t j = s ? i - c.n[0] : i;
        const uint64_t *off = s ? c.off[1] : c.off[0];
        const uint64_t p = (s ? c.p0[1] : c.p0[0]) + j;
        uint64_t lo = 0, hi = s ? c.n_off[1] : c.n_off[0];  // upper_bound(off, p) - 1 = the entry's genome in the slice
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (off[mid] > p) hi = mid; else lo = mid + 1;
        }
        const uint64_t genome = (s ? c.g0[1] : c.g0[0]) + lo - 1;
        const uint64_t key = s ? c.keys[1][j] : c.keys[0][j];
        const uint32_t at = atomicAdd(slot + bucket_of(key, M, NB) + 1, 1u);
        keys[at] = key;
        gid[at] = (uint32_t)(genome << 1) | (s ? c.part[1] : c.part[0]);
    }
}

constexpr uint32_t DB_SMALL = 16;   // buckets up to this size are sorted by one thread
constexpr uint32_t DB_MID = 2048;   // up to this size by one block in shared memory; larger ones one at a time (db_sort_large)
constexpr uint32_t DB_SORT_TILE = 256;

// Sorts every bucket of up to DB_MID entries in place by (key, tracked, genome) and lists the larger ones in large[]
// as (start, size).  Block i looks at buckets DB_SORT_TILE * i ..: a thread per small bucket, then the block on each
// middle-sized one (bitonic sort of the bucket padded to a power of two with entries above every real one).
__global__ void __launch_bounds__(DB_SORT_TILE) k_db_sort_buckets(const uint32_t *__restrict__ bstart, uint64_t NB,
                                                                  uint64_t *__restrict__ keys, uint32_t *__restrict__ gid,
                                                                  uint2 *__restrict__ large, unsigned long long *__restrict__ n_large) {
    __shared__ uint64_t sk[DB_MID];
    __shared__ uint32_t sr[DB_MID];
    __shared__ uint32_t mid_b[DB_SORT_TILE];
    __shared__ uint32_t n_mid;
    if (threadIdx.x == 0) n_mid = 0;
    __syncthreads();
    const uint64_t b = (uint64_t)blockIdx.x * DB_SORT_TILE + threadIdx.x;
    if (b < NB) {
        const uint32_t s = bstart[b], m = bstart[b + 1] - s;
        if (m > DB_MID) {
            large[atomicAdd(n_large, 1ull)] = make_uint2(s, m);
        } else if (m > DB_SMALL) {
            mid_b[atomicAdd(&n_mid, 1u)] = (uint32_t)(b - (uint64_t)blockIdx.x * DB_SORT_TILE);
        } else if (m > 1) {
            uint64_t k[DB_SMALL];
            uint32_t r[DB_SMALL];
            for (uint32_t i = 0; i < m; i++) {  // insertion sort
                const uint64_t ki = keys[s + i];
                const uint32_t ri = gid_rank(gid[s + i]);
                uint32_t j = i;
                for (; j > 0 && entry_less(ki, ri, k[j - 1], r[j - 1]); j--) { k[j] = k[j - 1]; r[j] = r[j - 1]; }
                k[j] = ki;
                r[j] = ri;
            }
            for (uint32_t i = 0; i < m; i++) { keys[s + i] = k[i]; gid[s + i] = rank_gid(r[i]); }
        }
    }
    __syncthreads();
    const uint32_t nm = n_mid;
    for (uint32_t q = 0; q < nm; q++) {
        const uint64_t bb = (uint64_t)blockIdx.x * DB_SORT_TILE + mid_b[q];
        const uint32_t s = bstart[bb], m = bstart[bb + 1] - s;
        uint32_t P = 32;
        while (P < m) P <<= 1;
        for (uint32_t i = threadIdx.x; i < P; i += DB_SORT_TILE) {
            sk[i] = i < m ? keys[s + i] : ~0ull;
            sr[i] = i < m ? gid_rank(gid[s + i]) : ~0u;  // real ranks are < 2^32 - 1
        }
        __syncthreads();
        for (uint32_t kk = 2; kk <= P; kk <<= 1) {
            for (uint32_t jj = kk >> 1; jj > 0; jj >>= 1) {
                for (uint32_t i = threadIdx.x; i < P; i += DB_SORT_TILE) {
                    const uint32_t x = i ^ jj;
                    if (x > i) {
                        const bool up = (i & kk) == 0;
                        if (entry_less(sk[x], sr[x], sk[i], sr[i]) == up) {
                            const uint64_t tk = sk[i]; sk[i] = sk[x]; sk[x] = tk;
                            const uint32_t tr = sr[i]; sr[i] = sr[x]; sr[x] = tr;
                        }
                    }
                }
                __syncthreads();
            }
        }
        for (uint32_t i = threadIdx.x; i < m; i += DB_SORT_TILE) { keys[s + i] = sk[i]; gid[s + i] = rank_gid(sr[i]); }
        __syncthreads();
    }
}

__global__ void k_gid_to_rank(const uint32_t *__restrict__ gid, uint32_t m, uint32_t *__restrict__ r) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) r[i] = gid_rank(gid[i]);
}

__global__ void k_rank_to_gid(const uint32_t *__restrict__ r, uint32_t m, uint32_t *__restrict__ gid) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) gid[i] = rank_gid(r[i]);
}

// SYL_ERR_ARG-worthy device offsets: off[0] != 0 or a decrease
__global__ void k_check_offsets(const uint64_t *__restrict__ off, uint64_t n, unsigned long long *__restrict__ bad) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (i == 0 ? off[0] != 0 : off[i] < off[i - 1])) *bad = 1ull;
}

// ---- the join -------------------------------------------------------------------------------
struct SampleView {
    const uint64_t *hash;
    const uint32_t *count;
    uint64_t n;
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
constexpr uint32_t COV_BINS = 256;

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

constexpr int BOOT_ITERS = 100;
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
// count >= COV_BINS or more rows than the table holds is reported in the header; contain_fast then
// redoes the call in the CSR formulation or with a larger table.
// CSR formulation (single GPU only): k_join_hist<probe only> records the equal ranges and
// k_join2_order<.., CSR_*> walks them twice per pass (count hits per pair, CUB scan, scatter the hits'
// sample counts), with no winner in pass 1; k_stats replaces k_stats_hist; ranking, bootstrap and finish
// are shared.  Sizing the value array after the pass-1 scan costs a second host synchronisation; pass 2
// needs none, because its hits are a subset of pass 1's (same ranges, winners only).
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

}  // namespace syl

namespace syl {
// what -u needs to know about a sample (src/contain.rs:377-408)
struct SampleMeta { double mean_read_length; uint64_t c, sum_counts; };

// Device bytes of one result row in the joins: two row tables, the bootstrap's results and its histogram
constexpr uint64_t ROW_BYTES = 2 * sizeof(syl_ani_row) + BOOT_ITERS * 17 + 17 * 4 + 8;

// What the joins of a host-sample batch may allocate beyond its plan (sample_batches.hpp charges neither): the CSR
// formulation's hit values (4 bytes per hit) and the row tables of a capacity retry.  The ctx's held plus transient
// device bytes stay within `limit` (0: unbounded, the handle path); a job that would pass it gives up with
// SPLIT_BATCH and contain_fast reruns its samples as two halves.  `want` is the refused allocation, `s0` the call's
// index of the job's first sample and `budget` the call's budget, for the error of a sample that does not fit alone.
struct JoinRoom {
    uint64_t limit = 0, budget = 0, want = 0;
    uint32_t s0 = 0;
};
constexpr int SPLIT_BATCH = -1;  // internal status, never returned through the C ABI

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
}

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
    bool csr = false;        // CSR formulation (single GPU) instead of the per-pair count histograms
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
};

namespace syl {

__global__ void k_sum_counts(const uint32_t *__restrict__ count, uint64_t n, unsigned long long *__restrict__ out) {
    unsigned long long acc = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) acc += count[i];
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

// Device handles as the views the joins take, and what -u needs to know of them (the sum of the counts is computed on the
// device once per handle, and only for -u).
static int handle_views(syl_ctx *ctx, const syl_sample *const *samples, uint32_t n, bool unknown, std::vector<SampleView> &views,
                        std::vector<SampleMeta> &metas) {
    cudaStream_t st = ctx->stream;
    views.resize(n);
    metas.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        syl_sample *s = const_cast<syl_sample *>(samples[i]);
        if (unknown && !s->sum_counts_valid) {
            unsigned long long *d = reinterpret_cast<unsigned long long *>(ctx->d_counters + CNT_SUM_COUNTS);
            SYL_CUDA(cudaMemsetAsync(d, 0, 8, st));
            if (s->n) k_sum_counts<<<ctx->num_sms * 4, 256, 0, st>>>(s->count, s->n, d);
            SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_SUM_COUNTS, d, 8, cudaMemcpyDeviceToHost, st));
            SYL_CUDA(cudaStreamSynchronize(st));
            s->sum_counts = ctx->h_counters[CNT_SUM_COUNTS];
            s->sum_counts_valid = true;
        }
        views[i] = {s->hash, s->count, s->n};
        metas[i] = {s->mean_read_length, s->c, s->sum_counts};
    }
    return SYL_OK;
}

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
// the walk on one GPU and from the all-reduced wbest across ranks (histogram formulation only).
template <JoinOut OUT>
static void join_walk(syl_profile_job *j, bool pass2) {
    const syl_db *db = j->db;
    if (!j->max_n || !db->N) return;
    auto k = k_join2_order<WIN_FUSED, OUT>;
    if constexpr (OUT == JOIN_HIST) {
        if (j->world > 1) k = k_join2_order<WIN_GIVEN, OUT>;
    } else {
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

// stage 1: allocate, pass 1 (P1 = the pass-1 parameters: profile skips the bootstrap there).  csr: the CSR formulation
// (single GPU only); otherwise histograms beyond 8 GB are SYL_ERR_UNSUPPORTED.
static int job_begin(syl_ctx *ctx, const syl_db *db, const SampleView *views, const SampleMeta *metas, uint32_t n_samples,
                     const syl_contain_params *p, bool profile, bool csr, uint32_t world, uint32_t rank, uint64_t R,
                     syl_profile_job **out, JoinRoom *room = nullptr) {
    cudaStream_t st = ctx->stream;
    Handle<syl_profile_job> h(new (std::nothrow) syl_profile_job());
    if (!h) return SYL_ERR_OOM;
    syl_profile_job *j = h.get();
    j->ctx = ctx; j->db = db; j->profile = profile; j->csr = csr; j->S = n_samples; j->G = db->n_genomes; j->world = world; j->rank = rank;
    j->room = room;
    syl_contain_params pp = *p;
    pp.pseudotax = profile ? 1 : 0;
    j->P = make_params(&pp);
    j->redundant_ani = pp.redundant_ani;
    if (p->estimate_unknown) { j->read_seq_id = p->read_seq_id; j->metas.assign(metas, metas + n_samples); }
    j->R = R ? ((R + 255) & ~255ull) : default_rows_per_rank(n_samples, db->n_genomes, world);
    j->tbytes = table_bytes(j->R);
    if (j->R * BOOT_ITERS >= 0xFFFF0000ull) { set_error("row capacity too large for the bootstrap work counter"); return SYL_ERR_ARG; }
    const uint64_t NP = (uint64_t)j->S * j->G;
    if (NP >= 0x7FFFFFFFull) { set_error("samples x genomes exceeds 2^31 pairs per call; split the sample batch"); return SYL_ERR_ARG; }
    if (!csr && !histograms_fit(NP)) { set_error("pair histograms exceed 8 GB; split the sample batch"); return SYL_ERR_UNSUPPORTED; }
    std::vector<SampleView> hv(views, views + n_samples);
    for (const SampleView &v : hv) j->max_n = std::max<uint64_t>(j->max_n, v.n);
    const uint64_t HN = std::max<uint64_t>((uint64_t)j->S * j->max_n, 1);
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
    if (j->S > 1 && j->max_n && db->N && !tile_env_off) {
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
    if (j->max_n && db->N) {
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

// single-GPU driver of the stages for syl_query / syl_profile.  The CSR formulation is taken up front when
// SYL_CONTAIN_CSR is set (read per call) or the per-pair histograms would exceed 8 GB, and after a histogram
// run that met a count >= COV_BINS; a row table that is too small is redone with the size it needed.
// `overlap`, when given, runs once, after the first attempt's stages are enqueued and before its result is awaited (the
// host samples stage their next batch there).  `room` (host-sample batches) bounds what the joins allocate beyond the
// batch's plan: CSR hit values or a capacity retry's row tables that do not fit it rerun the samples as two halves on
// the same views, recursively, and a single sample that does not fit is SYL_ERR_OOM.
static int contain_fast(syl_ctx *ctx, const syl_db *db, const SampleView *views, const SampleMeta *metas, uint32_t n_samples,
                        const syl_contain_params *p, bool profile, std::vector<syl_ani_row> &out,
                        const std::function<int()> &overlap = {}, JoinRoom *room = nullptr) {
    uint64_t R = 0;
    bool csr = getenv("SYL_CONTAIN_CSR") != nullptr || !histograms_fit((uint64_t)n_samples * db->n_genomes);
    bool overlapped = false;
    for (int attempt = 0; attempt < 4; attempt++) {  // one formulation switch + capacity retries
        syl_profile_job *j = nullptr;
        int rc = job_begin(ctx, db, views, metas, n_samples, p, profile, csr, 1, 0, R, &j, room);
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
        static const bool dbg = getenv("SYL_DEBUG_TIMING") != nullptr;
        if (dbg)
            fprintf(stderr, "[join split] samples %u..%u: %llu bytes do not fit, halves of %u and %u samples\n", room->s0,
                    room->s0 + n_samples, (unsigned long long)room->want, h, n_samples - h);
        JoinRoom r0 = *room, r1 = *room;
        r1.s0 += h;
        std::vector<syl_ani_row> second;
        SYL_TRY(contain_fast(ctx, db, views, metas, h, p, profile, out, overlapped ? std::function<int()>() : overlap, &r0));
        SYL_TRY(contain_fast(ctx, db, views + h, metas + h, n_samples - h, p, profile, second, {}, &r1));
        for (syl_ani_row &r : second) {
            r.sample += h;
            out.push_back(r);
        }
        return SYL_OK;
    }
    return SYL_ERR_CAPACITY;
}

// k and c of one sample against a database of k-mer size k and sketch parameter c
static int check_sample_kc(int k, uint64_t c, int sk, uint64_t sc) {
    if (sk != k) {  // src/contain.rs:608-615 (log::error + exit(1))
        set_error("k parameter for reads != k parameter for genome");
        return SYL_ERR_ARG;
    }
    if (c < sc) {   // src/contain.rs:616-623
        set_error("c parameter for reads > c parameter for genome");
        return SYL_ERR_ARG;
    }
    return SYL_OK;
}

// The parameters of a query or profile call against a database of k-mer size k that has_tracked k-mers or not
static int check_params(int k, bool has_tracked, bool profile, const syl_contain_params *p) {
    if (p->k != k) { set_error("params.k != db k"); return SYL_ERR_ARG; }
    if (p->estimate_unknown && !(p->read_seq_id > 0.)) {
        set_error("-u without --read-seq-id: the automatic read-identity estimate depends on hash-map iteration order (src/contain.rs:901-951)");
        return SYL_ERR_UNSUPPORTED;
    }
    if (profile && !has_tracked) {  // src/contain.rs:231-234
        set_error("Attempting profiling, but the database was sketched with the --disable-profiling option");
        return SYL_ERR_ARG;
    }
    return SYL_OK;
}

// The arguments of a query or profile call against a database of k-mer size k and sketch parameter c that has_tracked
// k-mers or not; *n_rows is 0 once they are not NULL.
static int check_contain_args(syl_ctx *ctx, int k, uint64_t c, bool has_tracked, bool profile, const syl_sample *const *samples,
                              uint32_t n_samples, const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!ctx || !p || !n_rows || (n_samples && !samples) || (cap && !rows)) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *n_rows = 0;
    for (uint32_t i = 0; i < n_samples; i++) {
        if (!samples[i]) { set_error("NULL sample"); return SYL_ERR_ARG; }
        SYL_TRY(check_sample_kc(k, c, samples[i]->k, samples[i]->c));
    }
    return check_params(k, has_tracked, profile, p);
}

// the rows of a call into the caller's buffer of cap rows; *n_rows is their number even when they do not fit
static int copy_rows(const std::vector<syl_ani_row> &out, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    *n_rows = out.size();
    if (out.size() > cap) { set_error("row buffer too small"); return SYL_ERR_CAPACITY; }
    std::copy(out.begin(), out.end(), rows);
    return SYL_OK;
}

// ---- index build, host side -------------------------------------------------------------------

// A large temporary of the index build: allocated outside the ctx's block cache (counted in its peak while it lives)
// and returned to the driver once the ctx stream has drained, so the build leaves nothing but the index behind.
struct BuildBuf {
    syl_ctx *ctx;
    void *p = nullptr;
    size_t bytes = 0;
    explicit BuildBuf(syl_ctx *c) : ctx(c) {}
    BuildBuf(const BuildBuf &) = delete;
    BuildBuf &operator=(const BuildBuf &) = delete;
    ~BuildBuf() { release(); }
    int alloc(size_t b) {
        release();
        b = (std::max<size_t>(b, 1) + 255) & ~(size_t)255;
        cudaError_t e = cudaMalloc(&p, b);
        if (e != cudaSuccess) {
            p = nullptr;
            set_error(std::string("cudaMalloc(") + std::to_string(b) + " B): " + cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? SYL_ERR_OOM : SYL_ERR_CUDA;
        }
        bytes = b;
        ctx->transient_bytes += b;
        note_device_bytes(ctx);
        return SYL_OK;
    }
    void release() {
        if (!p) return;
        cudaStreamSynchronize(ctx->stream);
        cudaFree(p);
        ctx->transient_bytes -= bytes;
        p = nullptr;
        bytes = 0;
    }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// The build's input: part 0 = genome k-mers, part 1 = tracked k-mers, each CSR over the same G genomes
// (off[part][0 .. G], validated: starts at 0, monotone).
struct DbInput {
    int mem;
    const uint64_t *keys[2], *off[2];
    uint64_t G, n[2];
};

static uint64_t db_chunk_entries() {  // SYL_DB_CHUNK overrides (tests; read per call)
    if (const char *e = getenv("SYL_DB_CHUNK")) {
        const long long v = atoll(e);
        if (v >= 1) return (uint64_t)v;
    }
    return 1ull << 25;
}

// Hands the input to a pass chunk by chunk.  A device source is one chunk over the whole arrays.  A host source is
// cut into chunks of at most C entries and, per segment, at most min(C, G) genome offsets; each chunk is copied on a
// second stream into one of two staging buffers while the previous chunk's kernels run on the ctx stream.
struct DbFeed {
    syl_ctx *ctx;
    const DbInput &in;
    uint64_t C = 0, L = 0;
    BuildBuf stage[2];
    cudaStream_t cs = nullptr;
    cudaEvent_t copied[2] = {}, done[2] = {};
    DbFeed(syl_ctx *c, const DbInput &i) : ctx(c), in(i), stage{BuildBuf(c), BuildBuf(c)} {}
    ~DbFeed() {
        cudaStreamSynchronize(ctx->stream);
        if (cs) { cudaStreamSynchronize(cs); cudaStreamDestroy(cs); }
        for (int b = 0; b < 2; b++) {
            if (copied[b]) cudaEventDestroy(copied[b]);
            if (done[b]) cudaEventDestroy(done[b]);
        }
    }
    int init() {
        if (in.mem == SYL_MEM_DEVICE) return SYL_OK;
        C = std::min<uint64_t>(db_chunk_entries(), in.n[0] + in.n[1]);
        L = std::min<uint64_t>(C, in.G);
        SYL_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) {
            SYL_CUDA(cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
            SYL_CUDA(cudaEventCreateWithFlags(&done[b], cudaEventDisableTiming));
            SYL_TRY(stage[b].alloc((C + 2 * L) * 8));
        }
        return SYL_OK;
    }
    // the host chunk that starts at entry e of the concatenated parts; advances e past it
    int plan(uint64_t &e, uint64_t p0[2], uint64_t p1[2], uint64_t glo[2], uint64_t ghi[2], uint32_t part[2]) const {
        uint64_t budget = C;
        int ns = 0;
        while (budget && e < in.n[0] + in.n[1] && ns < 2) {
            const uint32_t pt = e < in.n[0] ? 0 : 1;
            const uint64_t *off = in.off[pt];
            const uint64_t a = pt ? e - in.n[0] : e;
            const uint64_t g = (uint64_t)(std::upper_bound(off, off + in.G + 1, a) - off) - 1;
            uint64_t z = std::min(a + budget, in.n[pt]);
            if (g + L <= in.G) z = std::min(z, off[g + L]);  // > a: genome g holds entry a
            p0[ns] = a; p1[ns] = z; glo[ns] = g; part[ns] = pt;
            ghi[ns] = (uint64_t)(std::upper_bound(off, off + in.G + 1, z - 1) - off) - 1;
            ns++;
            budget -= z - a;
            e += z - a;
            if (z < in.n[pt]) break;  // the chunk ends inside this part
        }
        return ns;
    }
    template <typename F> int pass(F launch) {
        cudaStream_t st = ctx->stream;
        if (in.mem == SYL_MEM_DEVICE) {
            DbChunk c{};
            int ns = 0;
            for (uint32_t pt = 0; pt < 2; pt++) {
                if (!in.n[pt]) continue;
                c.keys[ns] = in.keys[pt]; c.off[ns] = in.off[pt]; c.n_off[ns] = in.G + 1;
                c.g0[ns] = 0; c.p0[ns] = 0; c.n[ns] = in.n[pt]; c.part[ns] = pt;
                ns++;
            }
            launch(c);
            ctx->launches++;
            SYL_CUDA(cudaGetLastError());
            return SYL_OK;
        }
        uint64_t e = 0;
        for (uint64_t i = 0; e < in.n[0] + in.n[1]; i++) {
            const int b = (int)(i & 1);
            uint64_t p0[2], p1[2], glo[2], ghi[2];
            uint32_t part[2];
            const int ns = plan(e, p0, p1, glo, ghi, part);
            if (i >= 2) SYL_CUDA(cudaStreamWaitEvent(cs, done[b], 0));
            uint64_t *kw = stage[b].as<uint64_t>(), *ow = kw + C;
            DbChunk c{};
            for (int s = 0; s < ns; s++) {
                const uint64_t n = p1[s] - p0[s], no = ghi[s] - glo[s] + 1;
                SYL_CUDA(cudaMemcpyAsync(kw, in.keys[part[s]] + p0[s], n * 8, cudaMemcpyHostToDevice, cs));
                SYL_CUDA(cudaMemcpyAsync(ow, in.off[part[s]] + glo[s], no * 8, cudaMemcpyHostToDevice, cs));
                c.keys[s] = kw; c.off[s] = ow; c.n_off[s] = no; c.g0[s] = glo[s]; c.p0[s] = p0[s]; c.n[s] = n; c.part[s] = part[s];
                kw += n;
                ow += no;
            }
            SYL_CUDA(cudaEventRecord(copied[b], cs));
            SYL_CUDA(cudaStreamWaitEvent(st, copied[b], 0));
            launch(c);
            ctx->launches++;
            SYL_CUDA(cudaGetLastError());
            SYL_CUDA(cudaEventRecord(done[b], st));
        }
        return SYL_OK;
    }
};

static unsigned db_grid(const syl_ctx *ctx, const DbChunk &c) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(nblk(c.n[0] + c.n[1], 256), (uint64_t)ctx->num_sms * 16));
}

// Buckets of more than DB_MID entries, one at a time: two stable radix sorts (by rank, then by key) through temporaries
// sized by the largest of them.
static int db_sort_large(syl_ctx *ctx, syl_db *db, const std::vector<uint2> &large) {
    cudaStream_t st = ctx->stream;
    uint32_t mmax = 0;
    for (const uint2 &l : large) mmax = std::max(mmax, l.y);
    size_t t1 = 0, t2 = 0;
    SYL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                             (const uint64_t *)nullptr, (uint64_t *)nullptr, mmax, 0, 32, st));
    SYL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                             (const uint32_t *)nullptr, (uint32_t *)nullptr, mmax, 0, 64, st));
    const size_t tb = std::max(t1, t2);
    const size_t kb = ((size_t)mmax * 8 + 255) & ~(size_t)255, rb = ((size_t)mmax * 4 + 255) & ~(size_t)255;
    BuildBuf buf(ctx);
    SYL_TRY(buf.alloc(kb + 2 * rb + tb));
    uint64_t *kalt = buf.as<uint64_t>();
    uint32_t *ra = reinterpret_cast<uint32_t *>(buf.as<uint8_t>() + kb), *rb2 = reinterpret_cast<uint32_t *>(buf.as<uint8_t>() + kb + rb);
    void *tmp = buf.as<uint8_t>() + kb + 2 * rb;
    for (const uint2 &l : large) {
        uint64_t *k = db->keys + l.x;
        uint32_t *g = db->gid + l.x;
        size_t t = tb;
        k_gid_to_rank<<<nblk(l.y, 256), 256, 0, st>>>(g, l.y, ra);
        SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, t, ra, rb2, k, kalt, l.y, 0, 32, st));
        t = tb;
        SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, t, kalt, k, rb2, ra, l.y, 0, 64, st));
        k_rank_to_gid<<<nblk(l.y, 256), 256, 0, st>>>(ra, l.y, g);
        ctx->launches += 4;
    }
    SYL_CUDA(cudaGetLastError());
    return SYL_OK;
}

static const char *const BAD_OFFSETS = "offsets must start at 0 and be monotone";

// CSR offsets of G genomes in host memory (tracked_off may be NULL): the chunk planner and the scatter's genome search
// walk them, so they must start at 0 and never decrease
static int check_host_offsets(const uint64_t *kmer_off, const uint64_t *tracked_off, uint64_t G) {
    for (const uint64_t *o : {kmer_off, tracked_off}) {
        if (!o) continue;
        bool bad = o[0] != 0;
        for (uint64_t i = 1; i <= G && !bad; i++) bad = o[i] < o[i - 1];
        if (bad) { set_error(BAD_OFFSETS); return SYL_ERR_ARG; }
    }
    return SYL_OK;
}

static int check_db_size(uint64_t nk, uint64_t nt, uint64_t G) {
    if (nk >= 0xFFFFFFFFull || nt >= 0xFFFFFFFFull || nk + nt >= 0xFFFFFFFFull) {
        set_error("db shard holds more than 2^32-2 k-mers; shard the database");
        return SYL_ERR_ARG;
    }
    if (G >= 0x7FFFFFFFull) { set_error("too many genomes in one db shard"); return SYL_ERR_ARG; }
    return SYL_OK;
}

// a half-built index: its kernels may still be writing it
void HandleFree::operator()(syl_db *db) const {
    cudaStreamSynchronize(db->stream);
    syl_db_free(db);
}

// The index of `in` (see "index build" above).  gn_size: G sizes in in.mem's memory, or NULL (zeros).
static int db_build(syl_ctx *ctx, const DbInput &in, const uint64_t *gn_size, int has_tracked, int k, uint64_t c,
                    uint32_t genome_base, syl_db **out) {
    cudaStream_t st = ctx->stream;
    const uint64_t G = in.G, N = in.n[0] + in.n[1];
    Handle<syl_db> db = new_handle<syl_db>(ctx);
    if (!db) return SYL_ERR_OOM;
    db->n_genomes = G;
    db->genome_base = genome_base;
    db->N = N;
    db->has_tracked = has_tracked;
    db->k = k;
    db->c = c;
    SYL_TRY(hblock_alloc(ctx, (void **)&db->keys, std::max<uint64_t>(N, 1) * 8));
    SYL_TRY(hblock_alloc(ctx, (void **)&db->gid, std::max<uint64_t>(N, 1) * 4));
    SYL_TRY(hblock_alloc(ctx, (void **)&db->glen, std::max<uint64_t>(G, 1) * 4));
    db->h_gn_size.assign(G, 0);
    std::vector<uint32_t> h_glen;
    if (G) {
        if (in.mem == SYL_MEM_DEVICE) {
            if (gn_size) SYL_CUDA(cudaMemcpyAsync(db->h_gn_size.data(), gn_size, G * 8, cudaMemcpyDeviceToHost, st));
            k_glen<<<nblk(G, 256), 256, 0, st>>>(in.off[0], G, db->glen);
            ctx->launches++;
        } else {
            if (gn_size) std::copy(gn_size, gn_size + G, db->h_gn_size.begin());
            h_glen.resize(G);
            for (uint64_t g = 0; g < G; g++) h_glen[g] = (uint32_t)(in.off[0][g + 1] - in.off[0][g]);
            SYL_CUDA(cudaMemcpyAsync(db->glen, h_glen.data(), G * 4, cudaMemcpyHostToDevice, st));
        }
    }
    uint64_t NB = 1024;
    while (NB < N / 4) NB <<= 1;
    db->NB = NB;
    SYL_TRY(hblock_alloc(ctx, (void **)&db->bstart, (NB + 2) * 4));
    SYL_CUDA(cudaMemsetAsync(db->bstart, 0, (NB + 2) * 4, st));
    if (N) {
        DbFeed feed(ctx, in);
        SYL_TRY(feed.init());
        unsigned long long *d_max = reinterpret_cast<unsigned long long *>(ctx->d_counters + CNT_MAX_KEY);
        SYL_CUDA(cudaMemsetAsync(d_max, 0, 16, st));  // CNT_MAX_KEY, CNT_LARGE_BUCKETS
        SYL_TRY(feed.pass([&](const DbChunk &ch) { k_db_max<<<db_grid(ctx, ch), 256, 0, st>>>(ch, d_max); }));
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_MAX_KEY, d_max, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        db->maxkey = ctx->h_counters[CNT_MAX_KEY];
        unsigned __int128 m = ((unsigned __int128)NB << 64) / ((unsigned __int128)db->maxkey + 1);
        db->M = m > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)m;
        const uint64_t M = db->M;
        SYL_TRY(feed.pass([&](const DbChunk &ch) { k_db_hist<<<db_grid(ctx, ch), 256, 0, st>>>(ch, M, NB, db->bstart); }));
        {
            BuildBuf tmp(ctx);
            size_t tb = 0;
            SYL_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, db->bstart, db->bstart, (int)(NB + 2), st));
            SYL_TRY(tmp.alloc(tb));
            SYL_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, tb, db->bstart, db->bstart, (int)(NB + 2), st));
            ctx->launches++;
        }
        SYL_TRY(feed.pass([&](const DbChunk &ch) {
            k_db_scatter<<<db_grid(ctx, ch), 256, 0, st>>>(ch, M, NB, db->bstart, db->keys, db->gid);
        }));
        // everything below reads the index only: the staging buffers go before the large-bucket temporaries come
        feed.stage[0].release();
        feed.stage[1].release();
        BuildBuf large(ctx);
        SYL_TRY(large.alloc((N / (DB_MID + 1) + 1) * sizeof(uint2)));
        unsigned long long *d_nl = reinterpret_cast<unsigned long long *>(ctx->d_counters + CNT_LARGE_BUCKETS);
        k_db_sort_buckets<<<nblk(NB, DB_SORT_TILE), DB_SORT_TILE, 0, st>>>(db->bstart, NB, db->keys, db->gid,
                                                                            large.as<uint2>(), d_nl);
        ctx->launches++;
        SYL_CUDA(cudaGetLastError());
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_LARGE_BUCKETS, d_nl, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        std::vector<uint2> h_large(ctx->h_counters[CNT_LARGE_BUCKETS]);
        if (!h_large.empty()) {
            SYL_CUDA(cudaMemcpyAsync(h_large.data(), large.p, h_large.size() * sizeof(uint2), cudaMemcpyDeviceToHost, st));
            SYL_CUDA(cudaStreamSynchronize(st));
            large.release();
            SYL_TRY(db_sort_large(ctx, db.get(), h_large));
        }
    }
    SYL_CUDA(cudaStreamSynchronize(st));
    *out = db.release();
    return SYL_OK;
}

}  // namespace syl

// A database in borrowed host arrays, cut into index shards (syl_db_shards_*).
struct syl_db_shards {
    syl_ctx *ctx = nullptr;
    const uint64_t *kmers = nullptr, *kmer_off = nullptr, *tracked = nullptr, *tracked_off = nullptr, *gn_size = nullptr;
    uint64_t G = 0;
    int k = 31;
    uint64_t c = 200;
    uint64_t cap = 0;             // entries per shard, and per survivor index of several samples
    uint64_t survivor_max = 0;    // entries of one sample's survivor index
    std::vector<uint64_t> first;  // shard i = genomes [first[i], first[i + 1])
    uint64_t calls = 0;
    struct {                      // the rows of the last call, when they did not fit the caller's buffer
        uint64_t call = 0;        // 0: nothing kept
        bool profile = false;
        syl_contain_params p{};
        std::vector<const void *> key;  // the samples of the call (handle pointers, or host arrays and their count)
        std::vector<syl_ani_row> rows;
    } kept;
    uint64_t *pinned = nullptr;   // staging of the survivor k-mers (grow-only)
    uint64_t pinned_n = 0;
};

namespace syl {

constexpr uint64_t PAIRS_PER_CALL = 1ull << 22;  // (sample, genome) pairs per join: 4 GB of per-pair histograms

// Entries per shard when the caller gives none: the device's free memory at 16 bytes per entry (the build's peak is
// about 14), after an eighth of it and the histograms of PAIRS_PER_CALL pairs are set aside for the joins.
static int default_shard_entries(uint64_t *out) {
    size_t free_b = 0, total_b = 0;
    SYL_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t budget = free_b - free_b / 8, joins = PAIRS_PER_CALL * COV_BINS * 4;
    const uint64_t e = budget > joins ? (budget - joins) / 16 : 0;
    *out = std::min<uint64_t>(std::max<uint64_t>(e, 1ull << 20), SHARD_MAX_ENTRIES);
    return SYL_OK;
}

static uint64_t shard_entries_env() {  // SYL_DB_SHARD_ENTRIES caps max_entries (tests; read per syl_db_shards_create)
    if (const char *e = getenv("SYL_DB_SHARD_ENTRIES")) {
        const long long v = atoll(e);
        if (v >= 1) return (uint64_t)v;
    }
    return 0;
}

static double ms_since(std::chrono::steady_clock::time_point t) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
}

// The index of genomes [a, b) straight from the borrowed host arrays; only the offsets are copied (rebased to 0).
static int shard_build(const syl_db_shards *s, uint64_t a, uint64_t b, syl_db **out) {
    const uint64_t G = b - a;
    std::vector<uint64_t> ko(G + 1), to(s->tracked_off ? G + 1 : 0);
    for (uint64_t i = 0; i <= G; i++) ko[i] = s->kmer_off[a + i] - s->kmer_off[a];
    for (uint64_t i = 0; i < to.size(); i++) to[i] = s->tracked_off[a + i] - s->tracked_off[a];
    const uint64_t nt = to.empty() ? 0 : to[G];
    const DbInput in{SYL_MEM_HOST,
                     {ko[G] ? s->kmers + s->kmer_off[a] : nullptr, nt ? s->tracked + s->tracked_off[a] : nullptr},
                     {ko.data(), to.empty() ? nullptr : to.data()}, G, {ko[G], nt}};
    return db_build(s->ctx, in, s->gn_size ? s->gn_size + a : nullptr, s->tracked_off ? 1 : 0, s->k, s->c, (uint32_t)a, out);
}

// ---- the samples of a call, batch by batch --------------------------------------------------------

// The samples of a call as the joins take them, in batches of samples [first[b], first[b + 1]): device handles (views
// into their own arrays) or host arrays staged batch by batch into device slots (HostSamples).
struct SampleSource {
    std::vector<SampleMeta> metas;  // per sample
    JoinRoom room;                  // what the joins of a batch may take beyond its plan (handles: unbounded)
    virtual ~SampleSource() = default;
    // the batches of a join against an index of G genomes
    virtual void batches(uint64_t G, std::vector<uint32_t> &first) const = 0;
    // the most samples x genomes of a survivor join from sample s0 on, and whether such a batch must end before sample i
    virtual uint64_t survivor_pairs(uint32_t) const { return PAIRS_PER_CALL; }
    virtual bool cut_before(uint32_t) const { return false; }
    // views of samples [s0, s1), inside one batch, ready for work enqueued on the ctx stream from now on
    virtual int views(uint32_t s0, uint32_t s1, std::vector<SampleView> &v) = 0;
    // stage samples [s0, s1) ahead of their views() (host samples), while the last views are joined
    virtual int prefetch(uint32_t, uint32_t) { return SYL_OK; }
    // the joins of the last views() are enqueued on the ctx stream
    virtual void done() {}
};

// Device handles: batches of at most PAIRS_PER_CALL pairs.
struct HandleSamples : SampleSource {
    std::vector<SampleView> all;
    void batches(uint64_t G, std::vector<uint32_t> &first) const override {
        const uint32_t S = (uint32_t)all.size();
        const uint32_t per = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(S, PAIRS_PER_CALL / std::max<uint64_t>(G, 1)));
        first.clear();
        for (uint32_t s0 = 0; s0 < S; s0 += per) first.push_back(s0);
        first.push_back(S);
    }
    int views(uint32_t s0, uint32_t s1, std::vector<SampleView> &v) override {
        v.assign(all.begin() + s0, all.begin() + s1);
        return SYL_OK;
    }
};

// Host samples (syl_host_samples), staged on the device batch by batch (sample_batches.hpp).  Two slots each hold one
// batch (hash, count and rebased offsets), filled on the ingest copy stream and sorted there by hash within each sample
// (one segmented sort per batch, into the slot or the shared second buffer, whichever it ends in), while the ctx stream
// joins the other slot.  Events order the two streams; the host waits only where the joins already do.
struct HostSamples : SampleSource {
    syl_ctx *ctx;
    const syl_host_samples *in;
    bool pinned_hash = false, pinned_count = false;
    std::vector<uint32_t> plan;  // batch b: samples [plan[b], plan[b + 1])
    uint64_t plan_G = 0;
    struct Slot {
        DevBuf<uint64_t> hash, off;
        DevBuf<uint32_t> count;
        std::vector<uint64_t> h_off;  // the slot's offsets, rebased to its first sample
        uint32_t s0 = 0, s1 = 0;
        bool full = false;
        cudaEvent_t staged = nullptr, used = nullptr;
    } slot[2];
    DevBuf<uint64_t> alt_hash;
    DevBuf<uint32_t> alt_count;
    DevBuf<uint8_t> tmp;
    cudaStream_t cs = nullptr;
    int cur = -1;  // slot of the last views()

    HostSamples(syl_ctx *c, const syl_host_samples *s) : ctx(c), in(s) {}
    ~HostSamples() override {
        if (cs) cudaStreamSynchronize(cs);  // the slots go back to the ctx cache, whose users run on the ctx stream
        for (Slot &sl : slot)
            for (cudaEvent_t e : {sl.staged, sl.used})
                if (e) cudaEventDestroy(e);
    }
    void batches(uint64_t, std::vector<uint32_t> &first) const override { first = plan; }
    uint32_t batch_of(uint32_t i) const { return (uint32_t)(std::upper_bound(plan.begin(), plan.end(), i) - plan.begin() - 1); }
    uint64_t survivor_pairs(uint32_t s0) const override {
        const uint32_t b = batch_of(s0);
        return std::min<uint64_t>(PAIRS_PER_CALL, std::max<uint64_t>(plan_G, 1) * (plan[b + 1] - plan[b]));
    }
    bool cut_before(uint32_t i) const override { return std::binary_search(plan.begin(), plan.end(), i); }
    int find(uint32_t s0, uint32_t s1) const {
        for (int k = 0; k < 2; k++)
            if (slot[k].full && slot[k].s0 <= s0 && s1 <= slot[k].s1) return k;
        return -1;
    }
    // slots and sort storage for the largest batch of the plan; the copy stream starts behind the ctx stream's work so far
    int init() {
        uint64_t kmers = 0, S = 0;
        size_t tb = 0;
        for (size_t b = 0; b + 1 < plan.size(); b++) {
            const uint64_t n = in->off[plan[b + 1]] - in->off[plan[b]], m = plan[b + 1] - plan[b];
            kmers = std::max(kmers, n);
            S = std::max(S, m);
            cub::DoubleBuffer<uint64_t> dk(nullptr, nullptr);
            cub::DoubleBuffer<uint32_t> dv(nullptr, nullptr);
            size_t t = 0;
            SYL_CUDA(cub::DeviceSegmentedSort::SortPairs(nullptr, t, dk, dv, (int)n, (int)m, (const uint64_t *)nullptr,
                                                         (const uint64_t *)nullptr, ctx->stream));
            tb = std::max(tb, t);
        }
        SYL_TRY(ingest_copy_stream(ctx, &cs));
        cudaStream_t st = ctx->stream;
        for (Slot &sl : slot) {
            SYL_TRY(sl.hash.alloc(kmers, st)); SYL_TRY(sl.count.alloc(kmers, st)); SYL_TRY(sl.off.alloc(S + 1, st));
            SYL_CUDA(cudaEventCreateWithFlags(&sl.staged, cudaEventDisableTiming));
            SYL_CUDA(cudaEventCreateWithFlags(&sl.used, cudaEventDisableTiming));
        }
        SYL_TRY(alt_hash.alloc(kmers, st)); SYL_TRY(alt_count.alloc(kmers, st)); SYL_TRY(tmp.alloc(tb, st));
        SYL_CUDA(cudaEventRecord(slot[0].used, st));  // cached blocks may still be in use by earlier work on the ctx stream
        SYL_CUDA(cudaStreamWaitEvent(cs, slot[0].used, 0));
        return SYL_OK;
    }
    // samples [s0, s1) into slot k, once the joins of its last batch are done
    int stage(int k, uint32_t s0, uint32_t s1) {
        if (!cs) SYL_TRY(init());
        Slot &sl = slot[k];
        SYL_CUDA(cudaStreamWaitEvent(cs, sl.used, 0));
        const uint64_t a = in->off[s0], n = in->off[s1] - a;
        sl.h_off.resize(s1 - s0 + 1);
        for (uint32_t i = s0; i <= s1; i++) sl.h_off[i - s0] = in->off[i] - a;
        SYL_TRY(ingest_copy(ctx, sl.off.p, sl.h_off.data(), sl.h_off.size() * 8, false));
        SYL_TRY(ingest_copy(ctx, sl.hash.p, in->hash + a, n * 8, pinned_hash));
        SYL_TRY(ingest_copy(ctx, sl.count.p, in->count + a, n * 4, pinned_count));
        if (n) {
            cub::DoubleBuffer<uint64_t> dk(sl.hash.p, alt_hash.p);
            cub::DoubleBuffer<uint32_t> dv(sl.count.p, alt_count.p);
            size_t tb = tmp.cap_bytes;
            SYL_CUDA(cub::DeviceSegmentedSort::SortPairs(tmp.p, tb, dk, dv, (int)n, (int)(s1 - s0), sl.off.p, sl.off.p + 1, cs));
            ctx->launches += 4;
            if (dk.selector) sl.hash.swap(alt_hash);
            if (dv.selector) sl.count.swap(alt_count);
        }
        SYL_CUDA(cudaEventRecord(sl.staged, cs));
        sl.s0 = s0;
        sl.s1 = s1;
        sl.full = true;
        return SYL_OK;
    }
    int prefetch(uint32_t s0, uint32_t s1) override {
        if (find(s0, s1) >= 0) return SYL_OK;
        return stage(cur < 0 ? 0 : 1 - cur, s0, s1);
    }
    int views(uint32_t s0, uint32_t s1, std::vector<SampleView> &v) override {
        int k = find(s0, s1);
        if (k < 0) {
            k = cur < 0 ? 0 : 1 - cur;
            SYL_TRY(stage(k, s0, s1));
        }
        const Slot &sl = slot[k];
        SYL_CUDA(cudaStreamWaitEvent(ctx->stream, sl.staged, 0));
        v.resize(s1 - s0);
        for (uint32_t i = s0; i < s1; i++) {
            const uint64_t o = sl.h_off[i - sl.s0];
            v[i - s0] = {sl.hash.p + o, sl.count.p + o, sl.h_off[i + 1 - sl.s0] - o};
        }
        cur = k;
        return SYL_OK;
    }
    void done() override {
        if (cur >= 0) cudaEventRecord(slot[cur].used, ctx->stream);
    }
};

// Every sample of `src` against db, in the batches of `first`: the next batch is staged while one is joined, and `then`
// (samples [then[0], then[1]), if given) while the last one is.  Rows appended with the call's sample indices.
static int join_batches(syl_ctx *ctx, const syl_db *db, SampleSource &src, const std::vector<uint32_t> &first,
                        const uint32_t *then, const syl_contain_params *p, bool profile, std::vector<syl_ani_row> &rows) {
    std::vector<SampleView> v;
    for (size_t b = 0; b + 1 < first.size(); b++) {
        const uint32_t s0 = first[b], s1 = first[b + 1];
        SYL_TRY(src.views(s0, s1, v));
        std::function<int()> next;
        if (b + 2 < first.size()) next = [&] { return src.prefetch(s1, first[b + 2]); };
        else if (then) next = [&] { return src.prefetch(then[0], then[1]); };
        std::vector<syl_ani_row> part;
        JoinRoom room = src.room;
        room.s0 = s0;
        const int rc = contain_fast(ctx, db, v.data(), src.metas.data() + s0, s1 - s0, p, profile, part, next, &room);
        src.done();
        SYL_TRY(rc);
        for (syl_ani_row &r : part) {
            r.sample += s0;
            rows.push_back(r);
        }
    }
    return SYL_OK;
}

// Pass 1 (syl_query) of every sample of src against every shard in turn: each shard's index is built once, joined with
// all samples batch by batch, and freed before the next one is built.  rows: by shard, then by (sample, genome);
// row.genome is the global index.
static int shards_sweep(syl_db_shards *s, SampleSource &src, const syl_contain_params *p, std::vector<syl_ani_row> &rows) {
    syl_ctx *ctx = s->ctx;
    std::vector<uint32_t> first, next;
    for (size_t i = 0; i + 1 < s->first.size(); i++) {
        const uint64_t a = s->first[i], G = s->first[i + 1] - a;
        // each shard's index and join scratch are allocated to that shard's size, not next to the previous shard's
        SYL_TRY(cache_trim(ctx));
        const auto t0 = std::chrono::steady_clock::now();
        syl_db *db = nullptr;
        SYL_TRY(shard_build(s, a, s->first[i + 1], &db));
        const double build_ms = ms_since(t0);
        const auto t1 = std::chrono::steady_clock::now();
        src.batches(G, first);
        next.clear();
        if (i + 2 < s->first.size()) src.batches(s->first[i + 2] - s->first[i + 1], next);
        const int rc = join_batches(ctx, db, src, first, next.size() > 1 ? next.data() : nullptr, p, false, rows);
        static const bool dbg = getenv("SYL_DEBUG_TIMING") != nullptr;
        if (dbg)
            fprintf(stderr, "[db shard %zu/%zu] genomes %llu+%llu entries %llu: build %.1f ms, pass 1 %.1f ms\n", i + 1,
                    s->first.size() - 1, (unsigned long long)a, (unsigned long long)G, (unsigned long long)db->N, build_ms, ms_since(t1));
        syl_db_free(db);
        SYL_TRY(rc);
    }
    return cache_trim(ctx);
}

// syl_profile of samples[s0, s1) of src on an index of the genomes `ids` (ascending global indices), gathered from the
// borrowed arrays into pinned staging; rows appended with global sample and genome indices.
static int survivor_profile(syl_db_shards *s, const std::vector<uint32_t> &ids, SampleSource &src, uint32_t s0, uint32_t s1,
                            const syl_contain_params *p, std::vector<syl_ani_row> &out) {
    const auto t0 = std::chrono::steady_clock::now();
    // host samples are staged on the copy stream while the index is gathered and built; the ctx stream waits for them
    // only before the joins (views() below)
    SYL_TRY(src.prefetch(s0, s1));
    const uint64_t n = ids.size();
    std::vector<uint64_t> ko(n + 1, 0), to(n + 1, 0), gsz(n, 0);
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t g = ids[i];
        ko[i + 1] = ko[i] + s->kmer_off[g + 1] - s->kmer_off[g];
        to[i + 1] = to[i] + s->tracked_off[g + 1] - s->tracked_off[g];
        if (s->gn_size) gsz[i] = s->gn_size[g];
    }
    const uint64_t nk = ko[n], nt = to[n];
    if (nk + nt > s->pinned_n) {
        if (s->pinned) cudaFreeHost(s->pinned);
        s->pinned = nullptr;
        s->pinned_n = 0;
        SYL_CUDA(cudaHostAlloc((void **)&s->pinned, (nk + nt) * 8, cudaHostAllocDefault));
        s->pinned_n = nk + nt;
    }
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t g = ids[i];
        std::copy(s->kmers + s->kmer_off[g], s->kmers + s->kmer_off[g + 1], s->pinned + ko[i]);
        std::copy(s->tracked + s->tracked_off[g], s->tracked + s->tracked_off[g + 1], s->pinned + nk + to[i]);
    }
    syl_db *db = nullptr;
    SYL_TRY(syl_db_build_arrays(s->ctx, SYL_MEM_HOST, s->pinned, ko.data(), s->pinned + nk, to.data(), gsz.data(), n, s->k,
                                s->c, 0, &db));
    const double build_ms = ms_since(t0);
    const auto t1 = std::chrono::steady_clock::now();
    std::vector<SampleView> v;
    std::vector<syl_ani_row> part;
    JoinRoom room = src.room;
    room.s0 = s0;
    int rc = src.views(s0, s1, v);
    if (rc == SYL_OK) rc = contain_fast(s->ctx, db, v.data(), src.metas.data() + s0, s1 - s0, p, true, part, {}, &room);
    src.done();
    syl_db_free(db);
    SYL_TRY(rc);
    static const bool dbg = getenv("SYL_DEBUG_TIMING") != nullptr;
    if (dbg)
        fprintf(stderr, "[survivor index] samples %u..%u genomes %llu entries %llu: gather+build %.1f ms, profile %.1f ms\n", s0, s1,
                (unsigned long long)n, (unsigned long long)(nk + nt), build_ms, ms_since(t1));
    for (syl_ani_row &r : part) {
        r.sample += s0;
        r.genome = ids[r.genome];
        out.push_back(r);
    }
    return SYL_OK;
}

// Profile over all shards, equal to syl_profile on one db of every genome: the winner table, pass 2, derep and the
// abundances only ever see pass-1 survivors (src/contain.rs:284-334, 410-430).  So pass 1 runs per shard, without CIs
// (never reported; the ANI gate comes before the bootstrap), and each batch of samples is profiled on an index of the
// union of its survivors.  Ascending global order keeps the winner table's lowest-index tie rule.  A batch closes when
// the union would pass the shard cap (or the source's pair or batch limits); one sample's survivors alone may take up
// to survivor_max entries.
static int shards_profile(syl_db_shards *s, SampleSource &src, const syl_contain_params *p, std::vector<syl_ani_row> &out) {
    const uint32_t S = (uint32_t)src.metas.size();
    syl_contain_params p1 = *p;
    p1.no_ci = 1;
    p1.estimate_unknown = 0;
    p1.read_seq_id = -1.;
    if (p1.minimum_ani < 0.) p1.minimum_ani = 95.;  // profile's gate in a query-mode pass (make_params)
    std::vector<std::vector<uint32_t>> surv(S);
    {
        std::vector<syl_ani_row> rows1;
        SYL_TRY(shards_sweep(s, src, &p1, rows1));
        for (const syl_ani_row &r : rows1) surv[r.sample].push_back(r.genome);
    }
    std::vector<uint8_t> in(s->G, 0);
    std::vector<uint32_t> ids;
    uint64_t entries = 0;
    uint32_t s0 = 0;
    auto flush = [&](uint32_t s1) -> int {
        if (!ids.empty()) {
            std::sort(ids.begin(), ids.end());
            SYL_TRY(survivor_profile(s, ids, src, s0, s1, p, out));
            SYL_TRY(cache_trim(s->ctx));
        }
        for (uint32_t g : ids) in[g] = 0;
        ids.clear();
        entries = 0;
        s0 = s1;
        return SYL_OK;
    };
    for (uint32_t i = 0; i < S; i++) {
        uint64_t own = 0, add = 0, addg = 0;
        for (uint32_t g : surv[i]) {
            const uint64_t e = genome_entries(s->kmer_off, s->tracked_off, g);
            own += e;
            if (!in[g]) { add += e; addg++; }
        }
        if (own > s->survivor_max) {
            set_error("the pass-1 survivors of sample " + std::to_string(i) + " hold " + std::to_string(own) +
                      " index entries, more than one survivor index takes (" + std::to_string(s->survivor_max) + ")");
            return SYL_ERR_UNSUPPORTED;
        }
        const uint64_t ng = ids.size() + addg;
        if (i > s0 && (entries + add > s->cap || ng > SHARD_MAX_GENOMES || (uint64_t)(i - s0 + 1) * ng > src.survivor_pairs(s0) ||
                       src.cut_before(i))) {
            SYL_TRY(flush(i));
            add = own;
        }
        for (uint32_t g : surv[i])
            if (!in[g]) { in[g] = 1; ids.push_back(g); }
        entries += add;
    }
    return flush(S);
}

// syl_query_shards / syl_profile_shards / syl_*_host_samples with shards, after the argument checks.  key: the samples
// of the call, as the rows of a SYL_ERR_CAPACITY call are kept under.
static int shards_call(syl_db_shards *s, SampleSource &src, const std::vector<const void *> &key, const syl_contain_params *p,
                       bool profile, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    const uint64_t call = ++s->calls;
    auto &kp = s->kept;
    const bool retry = kp.call && kp.call + 1 == call && kp.profile == profile && !memcmp(&kp.p, p, sizeof *p) && kp.key == key;
    std::vector<syl_ani_row> out;
    if (retry) out.swap(kp.rows);
    kp.call = 0;
    std::vector<syl_ani_row>().swap(kp.rows);
    kp.key.clear();
    if (!retry && s->G && !src.metas.empty()) {
        if (profile) {
            SYL_TRY(shards_profile(s, src, p, out));
        } else {
            SYL_TRY(shards_sweep(s, src, p, out));
            std::sort(out.begin(), out.end(), [](const syl_ani_row &a, const syl_ani_row &b) {
                return a.sample != b.sample ? a.sample < b.sample : a.genome < b.genome;
            });
        }
    }
    const int rc = copy_rows(out, rows, cap, n_rows);
    if (rc == SYL_ERR_CAPACITY) {
        kp.call = call;
        kp.profile = profile;
        kp.p = *p;
        kp.key = key;
        kp.rows.swap(out);
    }
    return rc;
}

static int handle_shards_call(syl_ctx *ctx, syl_db_shards *s, const syl_sample *const *samples, uint32_t n_samples,
                              const syl_contain_params *p, bool profile, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!s) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_TRY(check_contain_args(ctx, s->k, s->c, s->tracked_off != nullptr, profile, samples, n_samples, p, rows, cap, n_rows));
    if (ctx != s->ctx) { set_error("db shards used with another ctx than the one that created them"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    HandleSamples src;
    SYL_TRY(handle_views(ctx, samples, n_samples, p->estimate_unknown != 0, src.all, src.metas));
    return shards_call(s, src, std::vector<const void *>(samples, samples + n_samples), p, profile, rows, cap, n_rows);
}

// syl_query_host_samples / syl_profile_host_samples
static int host_samples_call(syl_ctx *ctx, const syl_db *db, syl_db_shards *sh, const syl_host_samples *s,
                             const syl_contain_params *p, bool profile, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!ctx || !s || !p || !n_rows || (cap && !rows)) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if ((db != nullptr) == (sh != nullptr)) { set_error("exactly one of db and shards must be given"); return SYL_ERR_ARG; }
    *n_rows = 0;
    const uint32_t S = s->n_samples;
    if (!s->off || (S && (!s->c || !s->mean_read_length))) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (s->off[0] != 0) { set_error(BAD_OFFSETS); return SYL_ERR_ARG; }
    for (uint32_t i = 0; i < S; i++)
        if (s->off[i + 1] < s->off[i]) { set_error(BAD_OFFSETS); return SYL_ERR_ARG; }
    if (s->off[S] && (!s->hash || !s->count)) { set_error("off counts k-mers but hash or count is NULL"); return SYL_ERR_ARG; }
    const int k = db ? db->k : sh->k;
    const uint64_t c = db ? db->c : sh->c;
    for (uint32_t i = 0; i < S; i++) SYL_TRY(check_sample_kc(k, c, s->k, s->c[i]));
    SYL_TRY(check_params(k, db ? db->has_tracked != 0 : sh->tracked_off != nullptr, profile, p));
    if (sh && ctx != sh->ctx) { set_error("db shards used with another ctx than the one that created them"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    HostSamples src(ctx, s);
    for (int a = 0; a < 2 && s->off[S]; a++) {  // pinned arrays are copied as they are, pageable ones through the ring
        cudaPointerAttributes at{};
        const void *ptr = a ? (const void *)s->count : (const void *)s->hash;
        bool pinned = false;
        if (cudaPointerGetAttributes(&at, ptr) == cudaSuccess) {
            if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) { set_error("host samples: a device pointer was given"); return SYL_ERR_ARG; }
            pinned = at.type == cudaMemoryTypeHost;
        } else {
            cudaGetLastError();
        }
        (a ? src.pinned_count : src.pinned_hash) = pinned;
    }
    // the plan: the device budget of syl_ctx_set_sample_memory (0: free memory once the ctx's staging ring exists, plus
    // the ctx's cached free blocks), less the largest shard's build (16 bytes per entry)
    cudaStream_t cs = nullptr;
    SYL_TRY(ingest_copy_stream(ctx, &cs));
    uint64_t budget = ctx->sample_budget, index = 0;
    if (!budget) {
        size_t free_b = 0, total_b = 0;
        SYL_CUDA(cudaMemGetInfo(&free_b, &total_b));
        budget = free_b;
        for (const auto &b : ctx->free_blocks) budget += b.second;
    }
    // the joins' allocations beyond the plan are held to the budget on top of the bytes the ctx holds in use now
    uint64_t live = ctx->cached_bytes + ctx->transient_bytes;
    for (const auto &b : ctx->free_blocks) live -= b.second;
    src.room.limit = live + budget;
    src.room.budget = budget;
    if (sh) {
        for (size_t i = 0; i + 1 < sh->first.size(); i++) {
            const uint64_t a = sh->first[i], b = sh->first[i + 1];
            src.plan_G = std::max(src.plan_G, b - a);
            index = std::max(index, 16 * (sh->kmer_off[b] - sh->kmer_off[a] + (sh->tracked_off ? sh->tracked_off[b] - sh->tracked_off[a] : 0)));
        }
    } else {
        src.plan_G = db->n_genomes;
    }
    uint32_t forced = 0;
    if (const char *e = getenv("SYL_SAMPLE_BATCH")) forced = (uint32_t)std::max(0, atoi(e));
    const BatchCost cost{36, 4 * 8 + sizeof(SampleView) + 96 * ROW_BYTES, 16, COV_BINS * 4 + 16, 256 * ROW_BYTES + (1u << 20)};
    uint32_t bad = 0;
    uint64_t need = 0;
    const BatchPlanResult pr = plan_sample_batches(s->off, S, src.plan_G, budget > index ? budget - index : 0, PAIRS_PER_CALL,
                                                   0x7FFFFFFFull, forced, cost, src.plan, &bad, &need);
    if (pr == BATCH_TOO_MANY_KMERS) {
        set_error("sample " + std::to_string(bad) + " holds " + std::to_string(need) + " k-mers, more than 2^31 - 1");
        return SYL_ERR_UNSUPPORTED;
    }
    if (pr == BATCH_OOM) {
        set_error("sample " + std::to_string(bad) + " needs " + std::to_string(need + index) + " bytes of device memory" +
                  (index ? " (with the largest shard's build)" : "") + ", the budget is " + std::to_string(budget) + " bytes");
        return SYL_ERR_OOM;
    }
    src.metas.resize(S);
    for (uint32_t i = 0; i < S; i++) {
        uint64_t sum = 0;
        if (p->estimate_unknown)
            for (uint64_t j = s->off[i]; j < s->off[i + 1]; j++) sum += s->count[j];
        src.metas[i] = {s->mean_read_length[i], s->c[i], sum};
    }
    if (sh) {
        const std::vector<const void *> key{s->hash, s->count, s->off, s->c, s->mean_read_length, (const void *)(uintptr_t)S};
        return shards_call(sh, src, key, p, profile, rows, cap, n_rows);
    }
    std::vector<syl_ani_row> out;
    if (db->n_genomes && S) SYL_TRY(join_batches(ctx, db, src, src.plan, nullptr, p, profile, out));
    return copy_rows(out, rows, cap, n_rows);
}

}  // namespace syl

using namespace syl;

extern "C" {

int syl_db_build(syl_ctx *ctx, const syl_genomes *g, uint32_t genome_base, syl_db **out) {
    if (!ctx || !g || !out) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_ENTER(ctx);
    const uint64_t nt = g->has_tracked ? g->total_tracked : 0;
    SYL_TRY(check_db_size(g->total_kmers, nt, g->n));
    const DbInput in{SYL_MEM_DEVICE, {g->kmers, g->tracked}, {g->kmer_off, g->tracked_off}, g->n, {g->total_kmers, nt}};
    return db_build(ctx, in, g->gn_size, g->has_tracked, g->k, g->c, genome_base, out);
}

int syl_db_build_arrays(syl_ctx *ctx, int mem, const uint64_t *kmers, const uint64_t *kmer_off, const uint64_t *tracked,
                        const uint64_t *tracked_off, const uint64_t *gn_size, uint64_t n_genomes, int k, uint64_t c,
                        uint32_t genome_base, syl_db **out) {
    if (!ctx || !kmer_off || !out) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    if (mem != SYL_MEM_HOST && mem != SYL_MEM_DEVICE) { set_error("bad mem"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    cudaStream_t st = ctx->stream;
    if (n_genomes >= 0x7FFFFFFFull) return check_db_size(0, 0, n_genomes);
    uint64_t nk = 0, nt = 0;
    if (mem == SYL_MEM_HOST) {
        nk = kmer_off[n_genomes];
        nt = tracked_off ? tracked_off[n_genomes] : 0;
    } else {
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_KMER_TOTAL, kmer_off + n_genomes, 8, cudaMemcpyDeviceToHost, st));
        if (tracked_off) SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_TRACKED_TOTAL, tracked_off + n_genomes, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        nk = ctx->h_counters[CNT_KMER_TOTAL];
        nt = tracked_off ? ctx->h_counters[CNT_TRACKED_TOTAL] : 0;
    }
    SYL_TRY(check_db_size(nk, nt, n_genomes));
    SYL_TRY(check_kmer_arrays(kmers, nk, tracked, nt));
    if (mem == SYL_MEM_HOST) {
        SYL_TRY(check_host_offsets(kmer_off, tracked_off, n_genomes));
    } else {
        unsigned long long *d_bad = reinterpret_cast<unsigned long long *>(ctx->d_counters + CNT_BAD_OFFSETS);
        SYL_CUDA(cudaMemsetAsync(d_bad, 0, 8, st));
        for (const uint64_t *o : {kmer_off, tracked_off}) {
            if (!o) continue;
            k_check_offsets<<<nblk(n_genomes + 1, 256), 256, 0, st>>>(o, n_genomes + 1, d_bad);
            ctx->launches++;
        }
        SYL_CUDA(cudaGetLastError());
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_BAD_OFFSETS, d_bad, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        if (ctx->h_counters[CNT_BAD_OFFSETS]) { set_error(BAD_OFFSETS); return SYL_ERR_ARG; }
    }
    const DbInput in{mem, {kmers, tracked}, {kmer_off, tracked_off}, n_genomes, {nk, nt}};
    return db_build(ctx, in, gn_size, tracked_off ? 1 : 0, k, c, genome_base, out);
}

int syl_db_download(syl_ctx *ctx, const syl_db *db, uint64_t *keys, uint32_t *gid, uint32_t *bstart, uint64_t *n_entries,
                    uint64_t *n_buckets) {
    if (!ctx || !db) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (n_entries) *n_entries = db->N;
    if (n_buckets) *n_buckets = db->NB;
    SYL_ENTER(ctx);
    cudaStream_t st = ctx->stream;
    if (keys && db->N) SYL_CUDA(cudaMemcpyAsync(keys, db->keys, db->N * 8, cudaMemcpyDeviceToHost, st));
    if (gid && db->N) SYL_CUDA(cudaMemcpyAsync(gid, db->gid, db->N * 4, cudaMemcpyDeviceToHost, st));
    if (bstart) SYL_CUDA(cudaMemcpyAsync(bstart, db->bstart, (db->NB + 1) * 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));
    return SYL_OK;
}

uint64_t syl_db_num_genomes(const syl_db *db) { return db ? db->n_genomes : 0; }

void syl_db_free(syl_db *db) {
    if (!db) return;
    cudaSetDevice(db->device);
    hblock_free(db->owner, db->keys);
    hblock_free(db->owner, db->gid);
    hblock_free(db->owner, db->bstart);
    hblock_free(db->owner, db->glen);
    delete db;
}

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

int syl_query(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
              const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!db) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_TRY(check_contain_args(ctx, db->k, db->c, db->has_tracked, false, samples, n_samples, p, rows, cap, n_rows));
    SYL_ENTER(ctx);
    if (db->n_genomes == 0 || n_samples == 0) return SYL_OK;
    std::vector<SampleView> views;
    std::vector<SampleMeta> metas;
    SYL_TRY(handle_views(ctx, samples, n_samples, p->estimate_unknown != 0, views, metas));
    std::vector<syl_ani_row> out;
    SYL_TRY(contain_fast(ctx, db, views.data(), metas.data(), n_samples, p, false, out));
    return copy_rows(out, rows, cap, n_rows);
}

int syl_profile_shard_begin(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                            const syl_contain_params *p, uint32_t world, uint32_t rank, uint64_t rows_per_rank,
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
    return job_begin(ctx, db, views.data(), metas.data(), n_samples, p, true, false, world, rank, rows_per_rank, out);
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

int syl_profile(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!db) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_TRY(check_contain_args(ctx, db->k, db->c, db->has_tracked, true, samples, n_samples, p, rows, cap, n_rows));
    SYL_ENTER(ctx);
    if (db->n_genomes == 0 || n_samples == 0) return SYL_OK;
    std::vector<SampleView> views;
    std::vector<SampleMeta> metas;
    SYL_TRY(handle_views(ctx, samples, n_samples, p->estimate_unknown != 0, views, metas));
    std::vector<syl_ani_row> out;
    SYL_TRY(contain_fast(ctx, db, views.data(), metas.data(), n_samples, p, true, out));
    return copy_rows(out, rows, cap, n_rows);
}

int syl_db_shards_create(syl_ctx *ctx, const uint64_t *kmers, const uint64_t *kmer_off, const uint64_t *tracked,
                         const uint64_t *tracked_off, const uint64_t *gn_size, uint64_t n_genomes, int k, uint64_t c,
                         uint64_t max_entries, syl_db_shards **out) {
    if (!ctx || !kmer_off || !out) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    if (n_genomes > 0xFFFFFFFFull) { set_error("more than 2^32 genomes: row.genome is 32 bits"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    for (const uint64_t *a : {kmers, kmer_off, tracked, tracked_off, gn_size}) {  // the sweep reads them on the host
        cudaPointerAttributes at{};
        if (!a) continue;
        if (cudaPointerGetAttributes(&at, a) != cudaSuccess) {
            cudaGetLastError();
            continue;
        }
        if (at.type == cudaMemoryTypeDevice) { set_error("db shards borrow host arrays; a device pointer was given"); return SYL_ERR_ARG; }
    }
    SYL_TRY(check_host_offsets(kmer_off, tracked_off, n_genomes));
    SYL_TRY(check_kmer_arrays(kmers, kmer_off[n_genomes], tracked, tracked_off ? tracked_off[n_genomes] : 0));
    uint64_t dflt = 0;
    SYL_TRY(default_shard_entries(&dflt));
    uint64_t cap = max_entries ? std::min(max_entries, SHARD_MAX_ENTRIES) : dflt;
    if (const uint64_t e = shard_entries_env()) cap = std::min(cap, e);
    std::vector<uint64_t> first;
    uint64_t big = 0;
    if (!cut_shards(kmer_off, tracked_off, n_genomes, cap, first, &big)) {
        set_error("genome " + std::to_string(big) + " alone holds more than 2^32-3 index entries");
        return SYL_ERR_ARG;
    }
    syl_db_shards *s = new (std::nothrow) syl_db_shards();
    if (!s) return SYL_ERR_OOM;
    s->ctx = ctx;
    s->kmers = kmers; s->kmer_off = kmer_off; s->tracked = tracked; s->tracked_off = tracked_off; s->gn_size = gn_size;
    s->G = n_genomes;
    s->k = k;
    s->c = c;
    s->cap = cap;
    s->survivor_max = std::max(cap, dflt);
    s->first.swap(first);
    *out = s;
    return SYL_OK;
}

uint64_t syl_db_shards_count(const syl_db_shards *s) { return s && !s->first.empty() ? s->first.size() - 1 : 0; }

int syl_db_shards_range(const syl_db_shards *s, uint64_t i, uint64_t *first_genome, uint64_t *n_genomes, uint64_t *n_entries) {
    if (!s || i >= syl_db_shards_count(s)) { set_error("NULL handle or shard index out of range"); return SYL_ERR_ARG; }
    const uint64_t a = s->first[i], b = s->first[i + 1];
    if (first_genome) *first_genome = a;
    if (n_genomes) *n_genomes = b - a;
    if (n_entries) *n_entries = s->kmer_off[b] - s->kmer_off[a] + (s->tracked_off ? s->tracked_off[b] - s->tracked_off[a] : 0);
    return SYL_OK;
}

int syl_query_shards(syl_ctx *ctx, syl_db_shards *s, const syl_sample *const *samples, uint32_t n_samples,
                     const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return handle_shards_call(ctx, s, samples, n_samples, p, false, rows, cap, n_rows);
}

int syl_profile_shards(syl_ctx *ctx, syl_db_shards *s, const syl_sample *const *samples, uint32_t n_samples,
                       const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return handle_shards_call(ctx, s, samples, n_samples, p, true, rows, cap, n_rows);
}

int syl_query_host_samples(syl_ctx *ctx, const syl_db *db, syl_db_shards *shards, const syl_host_samples *s,
                           const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return host_samples_call(ctx, db, shards, s, p, false, rows, cap, n_rows);
}

int syl_profile_host_samples(syl_ctx *ctx, const syl_db *db, syl_db_shards *shards, const syl_host_samples *s,
                             const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return host_samples_call(ctx, db, shards, s, p, true, rows, cap, n_rows);
}

void syl_db_shards_free(syl_db_shards *s) {
    if (!s) return;
    if (s->pinned) cudaFreeHost(s->pinned);
    delete s;
}

}  // extern "C"
