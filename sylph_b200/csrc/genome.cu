// genome.cu — genome (database) sketches from seeding survivors.
//
// Replaces sketch_genome (src/sketch.rs:550-622) and sketch_genome_individual (:481-548) for a
// batch of genomes:
//   (contig, pos, hash) tuples of all contigs        extract_markers_positions  :582 / :508
//   vec.sort()                                        :593 -> radix sort by (contig, pos)
//   k-mers seen >= 2x in the genome are dropped       :594-600,605 -> stable radix sort by hash:
//        equal hashes of one genome end up adjacent (genomes own contiguous contig ranges)
//   greedy min-spacing scan, per contig               :602-614 -> one thread per contig; the
//        reference's `last_contig != contig` reset makes every contig's chain independent and
//        its `last_pos == 0` sentinel can never collide with a real position (pos >= k-1)
//   kept -> genome_kmers, thinned -> pseudotax_tracked_nonused_kmers, both in position order
#include <cub/cub.cuh>

#include <new>
#include <vector>

#include "common.cuh"
#include "scan.cuh"

namespace syl {
int seed_device(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases, const uint64_t *d_rec_off,
                uint64_t off_bias, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos, syl_survivor *d_out,
                uint64_t cap, uint64_t *n_out);
}

namespace syl {

static inline unsigned nblk(uint64_t n, int bs) { return (unsigned)((n + bs - 1) / bs); }
static inline int bits_for(uint64_t maxval) {
    int b = 1;
    while (b < 64 && (maxval >> b)) b++;
    return b;
}

__global__ void k_split(const syl_survivor *__restrict__ sv, uint64_t n, uint64_t *__restrict__ key,
                        uint64_t *__restrict__ hash) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const syl_survivor s = sv[i];
    key[i] = ((uint64_t)s.rec << 32) | s.pos;
    hash[i] = s.hash;
}

__global__ void k_iota32(uint32_t *idx, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (uint32_t)i;
}

__global__ void k_iota64(uint64_t *v, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
}

// contig -> genome (upper_bound over genome_off)
__global__ void k_contig_genome(const uint64_t *__restrict__ genome_off, uint64_t n_genomes, uint64_t n_contigs,
                                uint32_t *__restrict__ cg) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_contigs) return;
    uint64_t lo = 0, hi = n_genomes + 1;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (genome_off[mid] > r) hi = mid; else lo = mid + 1;
    }
    cg[r] = (uint32_t)(lo - 1);
}

// hs/ix: survivors stably sorted by hash (ix = index into the position-sorted arrays).
// A hash occurring >= 2x inside one genome marks all its occurrences (src/sketch.rs:594-600).
__global__ void k_flag_dups(const uint64_t *__restrict__ hs, const uint32_t *__restrict__ ix, uint64_t n,
                            const uint64_t *__restrict__ poskey, const uint32_t *__restrict__ cg,
                            uint8_t *__restrict__ flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t h = hs[i];
    const uint32_t me = ix[i];
    const uint32_t g = cg[poskey[me] >> 32];
    bool dup = false;
    if (i > 0 && hs[i - 1] == h) dup |= cg[poskey[ix[i - 1]] >> 32] == g;
    if (i + 1 < n && hs[i + 1] == h) dup |= cg[poskey[ix[i + 1]] >> 32] == g;
    flag[me] = dup ? 0 : 3;  // 0 = duplicate (dropped); 3 = undecided, resolved by k_spacing
}

__device__ __forceinline__ uint64_t lower_bound_u64(const uint64_t *a, uint64_t n, uint64_t v) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Greedy min-spacing selection (src/sketch.rs:602-614): 1 = kept, 2 = tracked (thinned out).
// The reference walks a contig keeping a k-mer iff pos - last_kept > min_spacing.  A k-mer whose
// distance to the PREVIOUS non-duplicate k-mer already exceeds min_spacing is kept whatever
// happened before it (last_kept <= previous position), so the walk splits into independent
// clusters of closely spaced k-mers, each starting with such a head.  One thread per survivor:
// heads walk their (tiny: ~1.15 elements at c=200) cluster; everything else returns.
__global__ void k_spacing(const uint64_t *__restrict__ poskey, uint64_t n, uint64_t min_spacing,
                          uint8_t *__restrict__ flag, const uint32_t *__restrict__ d_n = nullptr) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d_n && *d_n < n) n = *d_n;
    if (i >= n || flag[i] == 0) return;
    const uint64_t key = poskey[i], contig = key >> 32, pos = key & 0xFFFFFFFFull;
    // previous non-duplicate survivor of the same contig
    bool head = true;
    for (uint64_t j = i; j-- > 0;) {
        const uint64_t kj = poskey[j];
        if ((kj >> 32) != contig) break;
        if (flag[j] == 0) continue;  // duplicates never change state, so this read races with nothing
        head = pos - (kj & 0xFFFFFFFFull) > min_spacing;
        break;
    }
    if (!head) return;
    flag[i] = 1;
    uint64_t last = pos, prev = pos;
    for (uint64_t k = i + 1; k < n; k++) {
        const uint64_t kk = poskey[k];
        if ((kk >> 32) != contig) break;
        if (flag[k] == 0) continue;
        const uint64_t pk = kk & 0xFFFFFFFFull;
        if (pk - prev > min_spacing) break;  // k is a head: its own thread takes over
        if (pk - last > min_spacing) { flag[k] = 1; last = pk; } else { flag[k] = 2; }
        prev = pk;
    }
}

struct FlagIs {
    uint8_t want;
    __host__ __device__ __forceinline__ FlagIs(uint8_t w) : want(w) {}
    __host__ __device__ __forceinline__ bool operator()(const uint8_t &f) const { return f == want; }
};

// per-genome CSR offsets: number of flag==want survivors before the genome's first survivor
__global__ void k_genome_offsets(const uint64_t *__restrict__ poskey, uint64_t n, const uint64_t *__restrict__ genome_off,
                                 uint64_t n_genomes, const uint64_t *__restrict__ scan_kept,
                                 const uint64_t *__restrict__ scan_tracked, uint64_t total_kept,
                                 uint64_t total_tracked, const uint64_t *__restrict__ contig_off,
                                 uint64_t *__restrict__ kmer_off, uint64_t *__restrict__ tracked_off,
                                 uint64_t *__restrict__ gn_size) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g > n_genomes) return;
    if (g == n_genomes) {
        kmer_off[g] = total_kept;
        tracked_off[g] = total_tracked;
        return;
    }
    const uint64_t first = lower_bound_u64(poskey, n, genome_off[g] << 32);
    kmer_off[g] = first < n ? scan_kept[first] : total_kept;
    tracked_off[g] = first < n ? scan_tracked[first] : total_tracked;
    gn_size[g] = contig_off[genome_off[g + 1]] - contig_off[genome_off[g]];  // src/sketch.rs:581
}

__global__ void k_scatter_flagged(const uint64_t *__restrict__ hash, const uint8_t *__restrict__ flag, uint64_t n,
                                  const uint64_t *__restrict__ scan_kept, const uint64_t *__restrict__ scan_tracked,
                                  uint64_t *__restrict__ kmers, uint64_t *__restrict__ tracked) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t f = flag[i];
    if (f == 1) kmers[scan_kept[i]] = hash[i];
    else if (f == 2 && tracked) tracked[scan_tracked[i]] = hash[i];
}

__global__ void k_flag_to_u64(const uint8_t *__restrict__ flag, uint64_t n, uint8_t want, uint64_t *__restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = flag[i] == want ? 1ull : 0ull;
}

__global__ void k_add_offset(const uint64_t *__restrict__ src, uint64_t n, uint64_t add, uint64_t *__restrict__ dst) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i] + add;
}

// block i copies genome i's k-mer and tracked ranges: src4 = {src_k, dst_k, src_t, dst_t} starts
__global__ void k_copy_ranges(const uint64_t *__restrict__ src4, const uint64_t *__restrict__ kmers,
                              const uint64_t *__restrict__ tracked, uint64_t *__restrict__ okmers,
                              uint64_t *__restrict__ otracked, const uint64_t *__restrict__ okoff,
                              const uint64_t *__restrict__ otoff) {
    const uint64_t i = blockIdx.x;
    const uint64_t sk = src4[4 * i], dk = src4[4 * i + 1], st = src4[4 * i + 2], dt = src4[4 * i + 3];
    const uint64_t nk = okoff[i + 1] - okoff[i], nt = otoff[i + 1] - otoff[i];
    for (uint64_t j = threadIdx.x; j < nk; j += blockDim.x) okmers[dk + j] = kmers[sk + j];
    for (uint64_t j = threadIdx.x; j < nt; j += blockDim.x) otracked[dt + j] = tracked[st + j];
}

// stream-ordered allocations on the creating ctx stream (no device-wide sync in steady-state loops)
static int genomes_alloc(syl_genomes *g, cudaStream_t st, uint64_t n_genomes, uint64_t nk, uint64_t nt) {
    g->stream = st;
    g->owner = tl_ctx;
    SYL_TRY(hblock_alloc(g->owner, (void **)&g->kmers, std::max<uint64_t>(nk, 1) * 8));
    SYL_TRY(hblock_alloc(g->owner, (void **)&g->tracked, std::max<uint64_t>(nt, 1) * 8));
    SYL_TRY(hblock_alloc(g->owner, (void **)&g->kmer_off, (n_genomes + 1) * 8));
    SYL_TRY(hblock_alloc(g->owner, (void **)&g->tracked_off, (n_genomes + 1) * 8));
    SYL_TRY(hblock_alloc(g->owner, (void **)&g->gn_size, std::max<uint64_t>(n_genomes, 1) * 8));
    g->n = n_genomes;
    g->total_kmers = nk;
    g->total_tracked = nt;
    return SYL_OK;
}

// Generic post-pass: two library radix sorts (position, then hash).  Handles every input; used when the
// slotted path below does not apply (tiny c, SYL_GENOME_POSTPASS=sort) or reports an overflow.
// Exactly one of d_bases (ASCII) / d_packed (2-bit words) is set, here and in the two functions below.
static int sketch_genomes_device_sort(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases,
                                      const uint64_t *d_contig_off, uint64_t n_contigs, const uint64_t *d_genome_off,
                                      uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax, int sem,
                                      syl_genomes *out) {
    cudaStream_t st = ctx->stream;
    // 1. survivors with positions
    uint64_t scap = n_bases / c + n_bases / (4 * c) + 65536;
    if (scap > n_bases) scap = n_bases + 16;
    DevBuf<syl_survivor> sv;
    uint64_t N = 0;
    for (;;) {
        SYL_TRY(sv.alloc(scap, st));
        int rc = seed_device(ctx, d_bases, d_packed, n_bases, d_contig_off, 0, n_contigs, k, c, sem, /*with_pos=*/1, sv.p, scap, &N);
        if (rc == SYL_ERR_CAPACITY) { scap = N + 16; continue; }
        if (rc != SYL_OK) return rc;
        break;
    }
    if (N >= 0xFFFFFFFFull) { set_error("more than 2^32-2 survivors in one genome batch; split the batch"); return SYL_ERR_ARG; }
    DevBuf<uint64_t> key_a, key_b, hash_a, hash_b, scan_k, scan_t;
    DevBuf<uint32_t> idx_a, idx_b, cg;
    DevBuf<uint8_t> flag, tmp;
    const uint64_t NA = std::max<uint64_t>(N, 1);
    SYL_TRY(key_a.alloc(NA, st)); SYL_TRY(key_b.alloc(NA, st));
    SYL_TRY(hash_a.alloc(NA, st)); SYL_TRY(hash_b.alloc(NA, st));
    SYL_TRY(idx_a.alloc(NA, st)); SYL_TRY(idx_b.alloc(NA, st));
    SYL_TRY(scan_k.alloc(NA, st)); SYL_TRY(scan_t.alloc(NA, st));
    SYL_TRY(flag.alloc(NA, st));
    SYL_TRY(cg.alloc(n_contigs, st));
    k_contig_genome<<<nblk(n_contigs, 256), 256, 0, st>>>(d_genome_off, n_genomes, n_contigs, cg.p);
    ctx->launches++;
    uint64_t total_kept = 0, total_tracked = 0;
    KernelTimer kt_post(ctx, SYL_KERNEL_GENOME_POST);
    if (N) {
        k_split<<<nblk(N, 256), 256, 0, st>>>(sv.p, N, key_a.p, hash_a.p);
        // 2. position order: sort by (contig, pos)
        const int pos_bits = 32 + bits_for(n_contigs);
        const int hash_bits = bits_for(fmh_threshold(c));
        size_t t1 = 0, t2 = 0, t3 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, t1, key_a.p, key_b.p, hash_a.p, hash_b.p, N, 0, pos_bits, st);
        cub::DeviceRadixSort::SortPairs(nullptr, t2, hash_b.p, hash_a.p, idx_a.p, idx_b.p, N, 0, hash_bits, st);
        cub::DeviceScan::ExclusiveSum(nullptr, t3, scan_k.p, scan_k.p, N, st);
        size_t tb = std::max(t1, std::max(t2, t3));
        SYL_TRY(tmp.alloc(tb, st));
        SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, key_a.p, key_b.p, hash_a.p, hash_b.p, N, 0, pos_bits, st));
        // now: key_b = poskey sorted, hash_b = hashes in position order
        // 3. duplicates inside a genome: stable sort of (hash, position index) by hash
        k_iota32<<<nblk(N, 256), 256, 0, st>>>(idx_a.p, N);
        tb = std::max(t1, std::max(t2, t3));
        SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, hash_b.p, hash_a.p, idx_a.p, idx_b.p, N, 0, hash_bits, st));
        k_flag_dups<<<nblk(N, 256), 256, 0, st>>>(hash_a.p, idx_b.p, N, key_b.p, cg.p, flag.p);
        // 4. greedy spacing per contig
        k_spacing<<<nblk(N, 256), 256, 0, st>>>(key_b.p, N, min_spacing, flag.p);
        // 5. compaction
        k_flag_to_u64<<<nblk(N, 256), 256, 0, st>>>(flag.p, N, 1, scan_k.p);
        k_flag_to_u64<<<nblk(N, 256), 256, 0, st>>>(flag.p, N, 2, scan_t.p);
        uint64_t *d_last = ctx->d_counters + 4;  // [4],[5]: last flags, [6],[7]: last scans
        SYL_CUDA(cudaMemcpyAsync(d_last, scan_k.p + (N - 1), 8, cudaMemcpyDeviceToDevice, st));
        SYL_CUDA(cudaMemcpyAsync(d_last + 1, scan_t.p + (N - 1), 8, cudaMemcpyDeviceToDevice, st));
        tb = std::max(t1, std::max(t2, t3));
        SYL_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, scan_k.p, scan_k.p, N, st));
        tb = std::max(t1, std::max(t2, t3));
        SYL_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, scan_t.p, scan_t.p, N, st));
        SYL_CUDA(cudaMemcpyAsync(d_last + 2, scan_k.p + (N - 1), 8, cudaMemcpyDeviceToDevice, st));
        SYL_CUDA(cudaMemcpyAsync(d_last + 3, scan_t.p + (N - 1), 8, cudaMemcpyDeviceToDevice, st));
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + 4, d_last, 32, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        total_kept = ctx->h_counters[4] + ctx->h_counters[6];
        total_tracked = ctx->h_counters[5] + ctx->h_counters[7];
        ctx->launches += 7 + 4;
    }
    out->has_tracked = pseudotax ? 1 : 0;
    if (!pseudotax) total_tracked = 0;
    SYL_TRY(genomes_alloc(out, st, n_genomes, total_kept, total_tracked));
    if (N) {
        k_scatter_flagged<<<nblk(N, 256), 256, 0, st>>>(hash_b.p, flag.p, N, scan_k.p, scan_t.p, out->kmers,
                                                         pseudotax ? out->tracked : nullptr);
        ctx->launches++;
    }
    k_genome_offsets<<<nblk(n_genomes + 1, 128), 128, 0, st>>>(key_b.p, N, d_genome_off, n_genomes, scan_k.p, scan_t.p,
                                                               total_kept, pseudotax ? total_tracked : 0, d_contig_off,
                                                               out->kmer_off, out->tracked_off, out->gn_size);
    ctx->launches++;
    kt_post.stop();
    SYL_CUDA(cudaGetLastError());
    if (!pseudotax) SYL_CUDA(cudaMemsetAsync(out->tracked_off, 0, (n_genomes + 1) * 8, st));
    SYL_CUDA(cudaStreamSynchronize(st));
    return SYL_OK;
}

// ------------------------------------------------------------------------------------------------
// Sort-free post-pass.
//   * k_seed writes every tile's survivors into the tile's own slot (SlotOut), so the output is in
//     tile = position order already; its flush orders the <= 512 survivors INSIDE a tile by
//     (contig, position) in shared memory and compacts the tiles (scan of the per-tile counts).
//   * duplicates (a hash seen twice in one genome, src/sketch.rs:594-600): a genome's survivors are now
//     contiguous; they are grouped through one L2-resident open-addressing table in which every genome
//     owns a region of twice its survivor count — no sort by hash, no per-CTA capacity to overflow.
//   * k_spacing as before; kept / tracked survivors are compacted with block counts + one small scan.
// One host synchronisation (the totals), like the read-sketch path.
constexpr uint32_t GEN_SLOT = 512;        // survivors per tile slot (= the seeding kernel's staging capacity)

// tile t: slot -> compact arrays at toff[t].  (Round 2 first ordered the slot here, by the rank of each survivor's
// window start in a 32 768-bit map of the tile; that ranking now runs inside k_seed's flush, where the survivors are
// still in shared memory, and this kernel is a copy.)
__global__ void __launch_bounds__(256)
k_tile_compact(const syl_survivor *__restrict__ slots, const uint32_t *__restrict__ tile_cnt, const uint32_t *__restrict__ toff,
               uint64_t n_tiles, uint64_t *__restrict__ poskey, uint64_t *__restrict__ hash) {
    // one warp per tile: the slot is already in position order (k_seed's slotted flush), so this is a copy
    const uint64_t t = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (t >= n_tiles) return;
    const uint32_t n = tile_cnt[t], out0 = toff[t];
    const syl_survivor *src = slots + t * GEN_SLOT;
    for (uint32_t i = threadIdx.x & 31; i < n; i += 32) {
        const syl_survivor sv = src[i];
        poskey[out0 + i] = ((uint64_t)sv.rec << 32) | sv.pos;
        hash[out0 + i] = sv.hash;
    }
}

// gs[g] = index of genome g's first survivor (g = 0 .. n_genomes; gs[n_genomes] = N); N from device memory
__global__ void k_genome_ranges(const uint64_t *__restrict__ poskey, const uint32_t *__restrict__ d_n, const uint64_t *__restrict__ genome_off,
                                uint64_t n_genomes, uint32_t *__restrict__ gs) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g > n_genomes) return;
    const uint64_t N = *d_n;
    gs[g] = g == n_genomes ? (uint32_t)N : (uint32_t)lower_bound_u64(poskey, N, genome_off[g] << 32);
}

// ---- duplicates (src/sketch.rs:594-600,605: a hash seen twice in one genome drops all its occurrences) ----
// One open-addressing table for the whole batch in global memory (blocks touch only their genomes' regions): genome g owns the
// slots [2 * gs[g], 2 * gs[g+1]) — load factor 1/2 whatever the genome's size or its share of repeats, so there is
// no table-overflow case.  A key is the 64-bit hash (< 2^63 for every c >= 2); bit 63 of a stored key is the
// "seen again" mark, set with an atomic OR by every later occurrence; the empty key is all ones.
constexpr unsigned long long DUP_EMPTY = 0xFFFFFFFFFFFFFFFFull, DUP_MARK = 1ull << 63;

// genome of survivor i: the last g with gs[g] <= i, searched between the genomes of the block's first and last
// survivor (s_lo / s_hi, found once per block)
__device__ __forceinline__ uint32_t dup_genome_of(const uint32_t *__restrict__ gs, uint64_t n_genomes, uint32_t i, uint32_t first, uint32_t last,
                                                   uint32_t *s_lo, uint32_t *s_hi) {
    if (threadIdx.x < 2) {
        const uint32_t x = threadIdx.x ? last : first;
        uint32_t lo = 0, hi = (uint32_t)n_genomes;
        while (lo + 1 < hi) { const uint32_t mid = (lo + hi) >> 1; if (gs[mid] <= x) lo = mid; else hi = mid; }
        *(threadIdx.x ? s_hi : s_lo) = lo;
    }
    __syncthreads();
    uint32_t lo = *s_lo, hi = *s_hi + 1;
    while (lo + 1 < hi) { const uint32_t mid = (lo + hi) >> 1; if (gs[mid] <= i) lo = mid; else hi = mid; }
    return lo;
}

__device__ __forceinline__ uint32_t dup_slot(unsigned long long h, uint32_t size) {
    return (uint32_t)((((h >> 6) & 0xFFFFFFFFull) * size) >> 32);  // hashes are uniform below the threshold: so are these 32 bits
}

__global__ void __launch_bounds__(256)
k_dups_insert(const uint64_t *__restrict__ hash, const uint32_t *__restrict__ gs, uint64_t n_genomes, const uint32_t *__restrict__ d_n,
              uint32_t cap, unsigned long long *__restrict__ table) {
    __shared__ uint32_t s_lo, s_hi;
    const uint32_t N = min(*d_n, cap), first = blockIdx.x * 256u;
    if (first >= N) return;
    const uint32_t i = first + threadIdx.x;
    const uint32_t g = dup_genome_of(gs, n_genomes, min(i, N - 1), first, min(first + 255u, N - 1), &s_lo, &s_hi);
    if (i >= N) return;
    const uint32_t base = gs[g], size = 2u * (gs[g + 1] - base);
    unsigned long long *T = table + 2ull * base;
    const unsigned long long h = hash[i];
    uint32_t sl = dup_slot(h, size);
    for (;;) {
        const unsigned long long prev = atomicCAS(&T[sl], DUP_EMPTY, h);
        if (prev == DUP_EMPTY) break;
        if ((prev & ~DUP_MARK) == h) { if (!(prev & DUP_MARK)) atomicOr(&T[sl], DUP_MARK); break; }
        if (++sl == size) sl = 0;
    }
}

// flag[i] = 0: the hash occurs >= 2x in its genome (dropped), 3: undecided (k_spacing decides kept / tracked)
__global__ void __launch_bounds__(256)
k_dups_flag(const uint64_t *__restrict__ hash, const uint32_t *__restrict__ gs, uint64_t n_genomes, const uint32_t *__restrict__ d_n,
            uint32_t cap, const unsigned long long *__restrict__ table, uint8_t *__restrict__ flag) {
    __shared__ uint32_t s_lo, s_hi;
    const uint32_t N = min(*d_n, cap), first = blockIdx.x * 256u;
    if (first >= N) return;
    const uint32_t i = first + threadIdx.x;
    const uint32_t g = dup_genome_of(gs, n_genomes, min(i, N - 1), first, min(first + 255u, N - 1), &s_lo, &s_hi);
    if (i >= N) return;
    const uint32_t base = gs[g], size = 2u * (gs[g + 1] - base);
    const unsigned long long *T = table + 2ull * base;
    const unsigned long long h = hash[i];
    uint32_t sl = dup_slot(h, size);
    unsigned long long k;
    while (((k = T[sl]) & ~DUP_MARK) != h) { if (++sl == size) sl = 0; }  // every hash was inserted: the walk ends
    flag[i] = (k & DUP_MARK) ? 0 : 3;
}

// per block of 1024 survivors: number of kept (flag 1) and tracked (flag 2) ones
__global__ void __launch_bounds__(256) k_flag_counts(const uint8_t *__restrict__ flag, const uint32_t *__restrict__ d_n,
                                                     uint32_t *__restrict__ bk, uint32_t *__restrict__ bt) {
    __shared__ uint32_t sk[8], st_[8];
    const uint64_t N = *d_n, base = (uint64_t)blockIdx.x * 1024;
    uint32_t ck = 0, ct = 0;
    for (int e = 0; e < 4; e++) {
        const uint64_t i = base + threadIdx.x + 256 * e;
        if (i < N) { const uint8_t f = flag[i]; ck += f == 1; ct += f == 2; }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { ck += __shfl_xor_sync(0xffffffffu, ck, d); ct += __shfl_xor_sync(0xffffffffu, ct, d); }
    if ((threadIdx.x & 31) == 0) { sk[threadIdx.x >> 5] = ck; st_[threadIdx.x >> 5] = ct; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t a = 0, b = 0;
        for (int w = 0; w < 8; w++) { a += sk[w]; b += st_[w]; }
        bk[blockIdx.x] = a;
        bt[blockIdx.x] = b;
    }
}

// scatter the kept / tracked hashes of one 1024-survivor block (in order) and record, per survivor, how many
// kept / tracked ones precede it (the per-genome CSR offsets are read from these)
__global__ void __launch_bounds__(1024) k_scatter_flagged_blocks(const uint64_t *__restrict__ hash, const uint8_t *__restrict__ flag,
                                                                 const uint32_t *__restrict__ d_n, const uint32_t *__restrict__ bk_off,
                                                                 const uint32_t *__restrict__ bt_off, uint64_t *__restrict__ kmers,
                                                                 uint64_t *__restrict__ tracked, uint32_t *__restrict__ scan_k,
                                                                 uint32_t *__restrict__ scan_t) {
    __shared__ uint32_t wk[32], wt[32];
    const uint64_t N = *d_n, i = (uint64_t)blockIdx.x * 1024 + threadIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint8_t f = i < N ? flag[i] : 0;
    const uint32_t mk = __ballot_sync(0xffffffffu, f == 1), mt = __ballot_sync(0xffffffffu, f == 2);
    if (lane == 0) { wk[wid] = __popc(mk); wt[wid] = __popc(mt); }
    __syncthreads();
    uint32_t pk = bk_off[blockIdx.x], pt = bt_off[blockIdx.x];
    for (int w = 0; w < wid; w++) { pk += wk[w]; pt += wt[w]; }
    pk += __popc(mk & ((1u << lane) - 1u));
    pt += __popc(mt & ((1u << lane) - 1u));
    if (i < N) {
        scan_k[i] = pk;
        scan_t[i] = pt;
        if (f == 1) kmers[pk] = hash[i];
        else if (f == 2 && tracked) tracked[pt] = hash[i];
    }
}

__global__ void k_genome_offsets32(const uint32_t *__restrict__ gs, const uint32_t *__restrict__ d_n, const uint64_t *__restrict__ genome_off,
                                   uint64_t n_genomes, const uint32_t *__restrict__ scan_k, const uint32_t *__restrict__ scan_t,
                                   const uint32_t *__restrict__ d_tot_k, const uint32_t *__restrict__ d_tot_t, int pseudotax,
                                   const uint64_t *__restrict__ contig_off, uint64_t *__restrict__ kmer_off,
                                   uint64_t *__restrict__ tracked_off, uint64_t *__restrict__ gn_size) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g > n_genomes) return;
    const uint32_t N = *d_n, first = gs[g];
    kmer_off[g] = first < N ? scan_k[first] : *d_tot_k;
    tracked_off[g] = pseudotax ? (first < N ? scan_t[first] : *d_tot_t) : 0;
    if (g < n_genomes) gn_size[g] = contig_off[genome_off[g + 1]] - contig_off[genome_off[g]];  // src/sketch.rs:581
}

// rc SYL_ERR_UNSUPPORTED: a slot / table overflowed — the caller takes the generic path
static int sketch_genomes_device_slots(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases,
                                       const uint64_t *d_contig_off, uint64_t n_contigs, const uint64_t *d_genome_off,
                                       uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax, int sem,
                                       syl_genomes *out) {
    cudaStream_t st = ctx->stream;
    const uint64_t n_tiles = seed_cta_tiles(n_bases);
    if (n_tiles * GEN_SLOT >= 0xFFFFFFFFull) { set_error("genome batch too large; split the batch"); return SYL_ERR_ARG; }
    const uint64_t cap = std::min<uint64_t>(n_tiles * GEN_SLOT, n_bases / c + n_bases / (4 * c) + 65536);  // compact survivors
    DevBuf<syl_survivor> slots;
    DevBuf<uint32_t> tile_cnt, toff, gs, bk, bt, bk_off, bt_off, scan_k, scan_t, t1, t2, flags32;
    DevBuf<uint64_t> poskey, hash, tmp_k, tmp_t;
    DevBuf<unsigned long long> dup_table;
    DevBuf<uint8_t> flag;
    SYL_TRY(slots.alloc(n_tiles * GEN_SLOT, st));
    SYL_TRY(tile_cnt.alloc(n_tiles, st)); SYL_TRY(toff.alloc(n_tiles + 1, st));
    SYL_TRY(flags32.alloc(2, st));  // [0] slot overflow, [1] unused
    SYL_CUDA(cudaMemsetAsync(flags32.p, 0, 8, st));
    SYL_CUDA(cudaMemsetAsync(ctx->d_counters, 0, 2 * sizeof(uint64_t), st));
    SeedJob job;
    job.d_bases = d_bases; job.d_packed = d_packed; job.n_bases = n_bases; job.d_rec_off = d_contig_off; job.off_bias = 0; job.n_rec = n_contigs;
    job.k = k; job.c = c; job.sem = sem; job.with_pos = 1; job.d_out = slots.p; job.cap = n_tiles * GEN_SLOT;
    job.d_count = reinterpret_cast<unsigned long long *>(ctx->d_counters);
    job.slot_cap = GEN_SLOT; job.d_tile_cnt = tile_cnt.p; job.d_slot_overflow = flags32.p;
    SYL_TRY(seed_enqueue(ctx, job));
    KernelTimer kt_post(ctx, SYL_KERNEL_GENOME_POST);
    SYL_TRY(scan_u32(ctx, tile_cnt.p, n_tiles, toff.p, t1, t2));   // toff[n_tiles] = N (device)
    const uint32_t *d_n = toff.p + n_tiles;
    SYL_TRY(poskey.alloc(cap, st)); SYL_TRY(hash.alloc(cap, st)); SYL_TRY(flag.alloc(cap, st));
    k_tile_compact<<<nblk(n_tiles, 8), 256, 0, st>>>(slots.p, tile_cnt.p, toff.p, n_tiles, poskey.p, hash.p);
    SYL_TRY(gs.alloc(n_genomes + 1, st));
    k_genome_ranges<<<nblk(n_genomes + 1, 256), 256, 0, st>>>(poskey.p, d_n, d_genome_off, n_genomes, gs.p);
    SYL_TRY(dup_table.alloc(2 * cap, st));
    SYL_CUDA(cudaMemsetAsync(dup_table.p, 0xFF, 2 * cap * sizeof(unsigned long long), st));
    k_dups_insert<<<nblk(cap, 256), 256, 0, st>>>(hash.p, gs.p, n_genomes, d_n, (uint32_t)cap, dup_table.p);
    k_dups_flag<<<nblk(cap, 256), 256, 0, st>>>(hash.p, gs.p, n_genomes, d_n, (uint32_t)cap, dup_table.p, flag.p);
    // N is only known on the device: size the element-wise grids for the capacity (threads past N return)
    k_spacing<<<nblk(cap, 256), 256, 0, st>>>(poskey.p, cap, min_spacing, flag.p, d_n);
    const uint64_t nb = (cap + 1023) / 1024;
    SYL_TRY(bk.alloc(nb, st)); SYL_TRY(bt.alloc(nb, st)); SYL_TRY(bk_off.alloc(nb + 1, st)); SYL_TRY(bt_off.alloc(nb + 1, st));
    SYL_TRY(scan_k.alloc(cap, st)); SYL_TRY(scan_t.alloc(cap, st)); SYL_TRY(tmp_k.alloc(cap, st)); SYL_TRY(tmp_t.alloc(cap, st));
    k_flag_counts<<<(unsigned)nb, 256, 0, st>>>(flag.p, d_n, bk.p, bt.p);
    SYL_TRY(scan_u32(ctx, bk.p, nb, bk_off.p, t1, t2));
    DevBuf<uint32_t> t3, t4;
    SYL_TRY(scan_u32(ctx, bt.p, nb, bt_off.p, t3, t4));
    k_scatter_flagged_blocks<<<(unsigned)nb, 1024, 0, st>>>(hash.p, flag.p, d_n, bk_off.p, bt_off.p, tmp_k.p, pseudotax ? tmp_t.p : nullptr,
                                                            scan_k.p, scan_t.p);
    ctx->launches += 8;
    // per-genome offsets go straight into the handle; the k-mer arrays need the totals first
    out->has_tracked = pseudotax ? 1 : 0;
    out->stream = st;
    out->owner = tl_ctx;
    out->n = n_genomes;
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->kmer_off, (n_genomes + 1) * 8));
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->tracked_off, (n_genomes + 1) * 8));
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->gn_size, std::max<uint64_t>(n_genomes, 1) * 8));
    k_genome_offsets32<<<nblk(n_genomes + 1, 128), 128, 0, st>>>(gs.p, d_n, d_genome_off, n_genomes, scan_k.p, scan_t.p, bk_off.p + nb,
                                                                 bt_off.p + nb, pseudotax, d_contig_off, out->kmer_off, out->tracked_off,
                                                                 out->gn_size);
    ctx->launches++;
    kt_post.stop();
    SYL_CUDA(cudaGetLastError());
    uint32_t *h32 = reinterpret_cast<uint32_t *>(ctx->h_counters + 4);
    SYL_CUDA(cudaMemcpyAsync(h32, flags32.p, 8, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpyAsync(h32 + 2, bk_off.p + nb, 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpyAsync(h32 + 3, bt_off.p + nb, 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpyAsync(h32 + 4, d_n, 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));  // the one synchronisation of the call
    if (h32[0] || h32[1] || h32[4] > cap) return SYL_ERR_UNSUPPORTED;
    const uint64_t total_kept = h32[2], total_tracked = pseudotax ? h32[3] : 0;
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->kmers, std::max<uint64_t>(total_kept, 1) * 8));
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->tracked, std::max<uint64_t>(total_tracked, 1) * 8));
    out->total_kmers = total_kept;
    out->total_tracked = total_tracked;
    if (total_kept) SYL_CUDA(cudaMemcpyAsync(out->kmers, tmp_k.p, total_kept * 8, cudaMemcpyDeviceToDevice, st));
    if (total_tracked) SYL_CUDA(cudaMemcpyAsync(out->tracked, tmp_t.p, total_tracked * 8, cudaMemcpyDeviceToDevice, st));
    return SYL_OK;
}

int sketch_genomes_device(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases,
                          const uint64_t *d_contig_off, uint64_t n_contigs, const uint64_t *d_genome_off, uint64_t n_genomes,
                          int k, uint64_t c, uint64_t min_spacing, int pseudotax, int sem, syl_genomes *out) {
    const char *e = getenv("SYL_GENOME_POSTPASS");  // "sort" forces the generic path (tests); read per call
    const bool force_sort = e && std::string(e) == "sort";
    // slots hold 512 survivors per 32K-base tile: c >= 96 keeps the expected number below 350
    if (!force_sort && c >= 96 && n_bases && n_contigs && n_genomes) {
        const int rc = sketch_genomes_device_slots(ctx, d_bases, d_packed, n_bases, d_contig_off, n_contigs, d_genome_off,
                                                   n_genomes, k, c, min_spacing, pseudotax, sem, out);
        if (rc != SYL_ERR_UNSUPPORTED) return rc;
        // a slot or table overflowed (low-complexity sequence): release what was allocated and take the generic path
        hblock_free(out->owner, out->kmer_off); hblock_free(out->owner, out->tracked_off); hblock_free(out->owner, out->gn_size);
        out->kmer_off = out->tracked_off = out->gn_size = nullptr;
    }
    return sketch_genomes_device_sort(ctx, d_bases, d_packed, n_bases, d_contig_off, n_contigs, d_genome_off, n_genomes, k, c,
                                      min_spacing, pseudotax, sem, out);
}

// packed: the input is 2-bit words (device or host memory); else ASCII
static int sketch_genomes_impl(syl_ctx *ctx, int mem, const uint8_t *bases, const uint32_t *packed, uint64_t n_bases,
                               const uint64_t *contig_off, uint64_t n_contigs, const uint64_t *genome_off, uint64_t n_genomes,
                               int k, uint64_t c, uint64_t min_spacing, int pseudotax, int individual, int sem,
                               syl_genomes **out) {
    if (!ctx || !out || (!bases && !packed && n_bases) || !contig_off || (!individual && !genome_off)) {
        set_error("NULL argument");
        return SYL_ERR_ARG;
    }
    if (c == 0) { set_error("c must be >= 1"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    DevBuf<uint8_t> hb;   // host memory: staged copies, alive until the call's last sync
    DevBuf<uint32_t> hp;
    DevBuf<uint64_t> hc, hg;
    const uint8_t *d_bases = bases;
    const uint32_t *d_packed = packed;
    const uint64_t *d_coff = contig_off, *d_goff = genome_off;
    if (individual) n_genomes = n_contigs;
    if (mem == SYL_MEM_HOST) {
        if (packed) {
            const uint64_t nw = (n_bases + 15) / 16;
            SYL_TRY(hp.alloc(nw + 16, st));
            if (nw) SYL_CUDA(cudaMemcpyAsync(hp.p, packed, nw * 4, cudaMemcpyHostToDevice, st));
            d_packed = hp.p;
        } else {
            SYL_TRY(hb.alloc(n_bases + 64, st));
            if (n_bases) SYL_CUDA(cudaMemcpyAsync(hb.p, bases, n_bases, cudaMemcpyHostToDevice, st));
            d_bases = hb.p;
        }
        SYL_TRY(hc.alloc(n_contigs + 1, st));
        SYL_CUDA(cudaMemcpyAsync(hc.p, contig_off, (n_contigs + 1) * 8, cudaMemcpyHostToDevice, st));
        d_coff = hc.p;
        if (!individual) {
            SYL_TRY(hg.alloc(n_genomes + 1, st));
            SYL_CUDA(cudaMemcpyAsync(hg.p, genome_off, (n_genomes + 1) * 8, cudaMemcpyHostToDevice, st));
            d_goff = hg.p;
        }
    } else if (mem != SYL_MEM_DEVICE) {
        set_error("bad mem");
        return SYL_ERR_ARG;
    }
    if (individual) {  // every record is its own genome (src/sketch.rs:481-548)
        SYL_TRY(hg.alloc(n_contigs + 1, st));
        k_iota64<<<nblk(n_contigs + 1, 256), 256, 0, st>>>(hg.p, n_contigs + 1);
        ctx->launches++;
        d_goff = hg.p;
    }
    syl_genomes *g = new (std::nothrow) syl_genomes();
    if (!g) return SYL_ERR_OOM;
    g->device = ctx->device;
    g->k = k;
    g->c = c;
    int rc = sketch_genomes_device(ctx, d_bases, d_packed, n_bases, d_coff, n_contigs, d_goff, n_genomes, k, c, min_spacing,
                                   pseudotax, sem, g);
    if (rc != SYL_OK) { syl_genomes_free(g); return rc; }
    *out = g;
    return SYL_OK;
}

}  // namespace syl

using namespace syl;

extern "C" {

int syl_sketch_genomes(syl_ctx *ctx, int mem, const uint8_t *bases, uint64_t n_bases,
                       const uint64_t *contig_off, uint64_t n_contigs, const uint64_t *genome_off,
                       uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax,
                       int individual, int sem, syl_genomes **out) {
    return sketch_genomes_impl(ctx, mem, bases, nullptr, n_bases, contig_off, n_contigs, genome_off, n_genomes, k, c,
                               min_spacing, pseudotax, individual, sem, out);
}

int syl_sketch_genomes_packed2(syl_ctx *ctx, int mem, const uint32_t *packed, uint64_t n_bases,
                               const uint64_t *contig_off, uint64_t n_contigs, const uint64_t *genome_off,
                               uint64_t n_genomes, int k, uint64_t c, uint64_t min_spacing, int pseudotax,
                               int individual, int sem, syl_genomes **out) {
    return sketch_genomes_impl(ctx, mem, nullptr, packed, n_bases, contig_off, n_contigs, genome_off, n_genomes, k, c,
                               min_spacing, pseudotax, individual, sem, out);
}

int syl_genomes_upload(syl_ctx *ctx, int mem, const uint64_t *kmers, const uint64_t *kmer_off,
                       const uint64_t *tracked, const uint64_t *tracked_off, const uint64_t *gn_size,
                       uint64_t n_genomes, int k, uint64_t c, syl_genomes **out) {
    if (!ctx || !out || !kmer_off) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    cudaMemcpyKind kind = mem == SYL_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    uint64_t nk = 0, nt = 0;
    if (mem == SYL_MEM_HOST) {
        nk = kmer_off[n_genomes];
        nt = tracked_off ? tracked_off[n_genomes] : 0;
    } else {
        SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + 8, kmer_off + n_genomes, 8, cudaMemcpyDeviceToHost, st));
        if (tracked_off) SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + 9, tracked_off + n_genomes, 8, cudaMemcpyDeviceToHost, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        nk = ctx->h_counters[8];
        nt = tracked_off ? ctx->h_counters[9] : 0;
    }
    syl_genomes *g = new (std::nothrow) syl_genomes();
    if (!g) return SYL_ERR_OOM;
    g->device = ctx->device; g->k = k; g->c = c;
    g->has_tracked = (tracked && tracked_off) ? 1 : 0;
    int rc = genomes_alloc(g, st, n_genomes, nk, nt);
    if (rc != SYL_OK) { syl_genomes_free(g); return rc; }
    auto fill = [&]() -> int {  // any failure below frees the handle and its blocks
        if (nk) SYL_CUDA(cudaMemcpyAsync(g->kmers, kmers, nk * 8, kind, st));
        SYL_CUDA(cudaMemcpyAsync(g->kmer_off, kmer_off, (n_genomes + 1) * 8, kind, st));
        if (g->has_tracked) {
            if (nt) SYL_CUDA(cudaMemcpyAsync(g->tracked, tracked, nt * 8, kind, st));
            SYL_CUDA(cudaMemcpyAsync(g->tracked_off, tracked_off, (n_genomes + 1) * 8, kind, st));
        } else {
            SYL_CUDA(cudaMemsetAsync(g->tracked_off, 0, (n_genomes + 1) * 8, st));
        }
        if (gn_size && n_genomes) SYL_CUDA(cudaMemcpyAsync(g->gn_size, gn_size, n_genomes * 8, kind, st));
        else if (n_genomes) SYL_CUDA(cudaMemsetAsync(g->gn_size, 0, n_genomes * 8, st));
        SYL_CUDA(cudaStreamSynchronize(st));
        return SYL_OK;
    };
    if ((rc = fill()) != SYL_OK) { syl_genomes_free(g); return rc; }
    *out = g;
    return SYL_OK;
}

int syl_genomes_concat(syl_ctx *ctx, const syl_genomes *const *parts, uint32_t n_parts, syl_genomes **out) {
    if (!ctx || !out || (n_parts && !parts)) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    uint64_t G = 0, nk = 0, nt = 0;
    for (uint32_t i = 0; i < n_parts; i++) {
        if (!parts[i]) { set_error("NULL part"); return SYL_ERR_ARG; }
        if (parts[i]->k != parts[0]->k || parts[i]->c != parts[0]->c || parts[i]->has_tracked != parts[0]->has_tracked) {
            set_error("parts disagree on k / c / has_tracked");
            return SYL_ERR_ARG;
        }
        G += parts[i]->n; nk += parts[i]->total_kmers; nt += parts[i]->total_tracked;
    }
    syl_genomes *g = new (std::nothrow) syl_genomes();
    if (!g) return SYL_ERR_OOM;
    g->device = ctx->device;
    if (n_parts) { g->k = parts[0]->k; g->c = parts[0]->c; g->has_tracked = parts[0]->has_tracked; }
    int rc = genomes_alloc(g, st, G, nk, nt);
    if (rc != SYL_OK) { syl_genomes_free(g); return rc; }
    uint64_t g0 = 0, k0 = 0, t0 = 0;
    auto fill = [&]() -> int {  // any failure below frees the handle and its blocks
    for (uint32_t i = 0; i < n_parts; i++) {
        const syl_genomes *p = parts[i];
        if (p->total_kmers) SYL_CUDA(cudaMemcpyAsync(g->kmers + k0, p->kmers, p->total_kmers * 8, cudaMemcpyDeviceToDevice, st));
        if (p->total_tracked) SYL_CUDA(cudaMemcpyAsync(g->tracked + t0, p->tracked, p->total_tracked * 8, cudaMemcpyDeviceToDevice, st));
        if (p->n) SYL_CUDA(cudaMemcpyAsync(g->gn_size + g0, p->gn_size, p->n * 8, cudaMemcpyDeviceToDevice, st));
        k_add_offset<<<nblk(p->n + 1, 256), 256, 0, st>>>(p->kmer_off, p->n + 1, k0, g->kmer_off + g0);
        k_add_offset<<<nblk(p->n + 1, 256), 256, 0, st>>>(p->tracked_off, p->n + 1, t0, g->tracked_off + g0);
        ctx->launches += 2;
        g0 += p->n; k0 += p->total_kmers; t0 += p->total_tracked;
    }
    if (n_parts == 0) {
        SYL_CUDA(cudaMemsetAsync(g->kmer_off, 0, 8, st));
        SYL_CUDA(cudaMemsetAsync(g->tracked_off, 0, 8, st));
    }
    SYL_CUDA(cudaGetLastError());
    SYL_CUDA(cudaStreamSynchronize(st));
    return SYL_OK;
    };
    if ((rc = fill()) != SYL_OK) { syl_genomes_free(g); return rc; }
    *out = g;
    return SYL_OK;
}

int syl_genomes_select(syl_ctx *ctx, const syl_genomes *g, const uint32_t *idx, uint32_t n, syl_genomes **out) {
    if (!ctx || !g || !out || (n && !idx)) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    std::vector<uint64_t> koff(g->n + 1), toff(g->n + 1), gs(std::max<uint64_t>(g->n, 1));
    SYL_CUDA(cudaMemcpyAsync(koff.data(), g->kmer_off, (g->n + 1) * 8, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpyAsync(toff.data(), g->tracked_off, (g->n + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (g->n) SYL_CUDA(cudaMemcpyAsync(gs.data(), g->gn_size, g->n * 8, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));
    std::vector<uint64_t> nko(n + 1, 0), nto(n + 1, 0), ngs(std::max<uint32_t>(n, 1)), src(4 * (uint64_t)std::max<uint32_t>(n, 1));
    for (uint32_t i = 0; i < n; i++) {
        if (idx[i] >= g->n) { set_error("genome index out of range"); return SYL_ERR_ARG; }
        const uint64_t a = idx[i];
        nko[i + 1] = nko[i] + (koff[a + 1] - koff[a]);
        nto[i + 1] = nto[i] + (toff[a + 1] - toff[a]);
        ngs[i] = gs[a];
        src[4 * i] = koff[a]; src[4 * i + 1] = nko[i]; src[4 * i + 2] = toff[a]; src[4 * i + 3] = nto[i];
    }
    syl_genomes *o = new (std::nothrow) syl_genomes();
    if (!o) return SYL_ERR_OOM;
    o->device = ctx->device; o->k = g->k; o->c = g->c; o->has_tracked = g->has_tracked;
    int rc = genomes_alloc(o, st, n, nko[n], nto[n]);
    if (rc != SYL_OK) { syl_genomes_free(o); return rc; }
    DevBuf<uint64_t> d_src;
    if ((rc = d_src.alloc(4 * (uint64_t)std::max<uint32_t>(n, 1), st)) != SYL_OK) { syl_genomes_free(o); return rc; }
    auto fill = [&]() -> int {  // any failure below frees the handle and its blocks
        SYL_CUDA(cudaMemcpyAsync(o->kmer_off, nko.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st));
        SYL_CUDA(cudaMemcpyAsync(o->tracked_off, nto.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st));
        if (n) {
            SYL_CUDA(cudaMemcpyAsync(o->gn_size, ngs.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
            SYL_CUDA(cudaMemcpyAsync(d_src.p, src.data(), (size_t)n * 32, cudaMemcpyHostToDevice, st));
            k_copy_ranges<<<n, 256, 0, st>>>(d_src.p, g->kmers, g->tracked, o->kmers,
                                             o->tracked, o->kmer_off, o->tracked_off);
            ctx->launches++;
            SYL_CUDA(cudaGetLastError());
        }
        SYL_CUDA(cudaStreamSynchronize(st));
        return SYL_OK;
    };
    if ((rc = fill()) != SYL_OK) { syl_genomes_free(o); return rc; }
    *out = o;
    return SYL_OK;
}

uint64_t syl_genomes_count(const syl_genomes *g) { return g ? g->n : 0; }
uint64_t syl_genomes_total_kmers(const syl_genomes *g) { return g ? g->total_kmers : 0; }
uint64_t syl_genomes_total_tracked(const syl_genomes *g) { return g ? g->total_tracked : 0; }
int syl_genomes_has_tracked(const syl_genomes *g) { return g ? g->has_tracked : 0; }
int syl_genomes_k(const syl_genomes *g) { return g ? g->k : 0; }
uint64_t syl_genomes_c(const syl_genomes *g) { return g ? g->c : 0; }

int syl_genomes_download(syl_ctx *ctx, const syl_genomes *g, uint64_t *kmers, uint64_t *kmer_off,
                         uint64_t *tracked, uint64_t *tracked_off, uint64_t *gn_size) {
    if (!ctx || !g) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_CUDA(cudaSetDevice(ctx->device));
    syl::tl_ctx = ctx;
    cudaStream_t st = ctx->stream;
    if (kmers && g->total_kmers) SYL_CUDA(cudaMemcpyAsync(kmers, g->kmers, g->total_kmers * 8, cudaMemcpyDeviceToHost, st));
    if (kmer_off) SYL_CUDA(cudaMemcpyAsync(kmer_off, g->kmer_off, (g->n + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (tracked && g->total_tracked) SYL_CUDA(cudaMemcpyAsync(tracked, g->tracked, g->total_tracked * 8, cudaMemcpyDeviceToHost, st));
    if (tracked_off) SYL_CUDA(cudaMemcpyAsync(tracked_off, g->tracked_off, (g->n + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (gn_size && g->n) SYL_CUDA(cudaMemcpyAsync(gn_size, g->gn_size, g->n * 8, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));
    return SYL_OK;
}

int syl_genomes_device_ptrs(const syl_genomes *g, const uint64_t **kmers, const uint64_t **kmer_off,
                            const uint64_t **tracked, const uint64_t **tracked_off, const uint64_t **gn_size) {
    if (!g) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if (kmers) *kmers = g->kmers;
    if (kmer_off) *kmer_off = g->kmer_off;
    if (tracked) *tracked = g->tracked;
    if (tracked_off) *tracked_off = g->tracked_off;
    if (gn_size) *gn_size = g->gn_size;
    return SYL_OK;
}

void syl_genomes_free(syl_genomes *g) {
    if (!g) return;
    cudaSetDevice(g->device);
    hblock_free(g->owner, g->kmers);  // back into the owning ctx's block cache
    hblock_free(g->owner, g->kmer_off);
    hblock_free(g->owner, g->tracked);
    hblock_free(g->owner, g->tracked_off);
    hblock_free(g->owner, g->gn_size);
    delete g;
}

}  // extern "C"
