// genome.cu — genome (database) sketches from seeding survivors.
//
// Replaces sketch_genome (src/sketch.rs:550-622) and sketch_genome_individual (:481-548) for a
// batch of genomes:
//   (contig, pos, hash) tuples of all contigs        extract_markers_positions  :582 / :508
//   vec.sort()                                        :593 -> survivors in (contig, pos) order, from one of two
//        front halves: k_seed's per-tile slots, already in position order (c >= 96), or seed_device and one
//        radix sort by (contig, pos) (every c; the fallback of the slotted one)
//   k-mers seen >= 2x in the genome are dropped       :594-600,605 -> one open-addressing table of survivor
//        indices in which every genome owns a region (genomes own contiguous contig ranges)
//   greedy min-spacing scan, per contig               :602-614 -> k_spacing; the reference's
//        `last_contig != contig` reset makes every contig's chain independent and its `last_pos == 0`
//        sentinel can never collide with a real position (pos >= k-1)
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

__global__ void k_iota64(uint64_t *v, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
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
                          uint8_t *__restrict__ flag, const uint32_t *__restrict__ d_n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (*d_n < n) n = *d_n;
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

// ------------------------------------------------------------------------------------------------
// Post-pass.  A front half puts the survivors in (contig, pos) order: the slotted one (k_seed's per-tile slots, no
// sort) when c >= 96, the sorted one (radix sort) otherwise and whenever the slotted one overflows.  The back half
// turns them into the CSR: duplicates through one table, k_spacing, kept / tracked survivors compacted with block
// counts + one small scan.  N lives in device memory; the back half makes one host synchronisation (the totals).
constexpr uint32_t GEN_SLOT = 512;        // survivors per tile slot (= the seeding kernel's staging capacity)

// tile t: slot -> compact arrays at toff[t] (entries at or past cap are dropped: the back half then reports N > cap).
// One warp per tile: k_seed's slotted flush already wrote the slot in position order, so this is a copy.
__global__ void __launch_bounds__(256)
k_tile_compact(const syl_survivor *__restrict__ slots, const uint32_t *__restrict__ tile_cnt, const uint32_t *__restrict__ toff,
               uint64_t n_tiles, uint32_t cap, uint64_t *__restrict__ poskey, uint64_t *__restrict__ hash) {
    const uint64_t t = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (t >= n_tiles) return;
    const uint32_t n = tile_cnt[t], out0 = toff[t];
    const syl_survivor *src = slots + t * GEN_SLOT;
    for (uint32_t i = threadIdx.x & 31; i < n && out0 + i < cap; i += 32) {
        const syl_survivor sv = src[i];
        poskey[out0 + i] = ((uint64_t)sv.rec << 32) | sv.pos;
        hash[out0 + i] = sv.hash;
    }
}

// gs[g] = index of genome g's first survivor (g = 0 .. n_genomes); gs[n_genomes] = min(N, cap), the count every
// later kernel of the back half works on
__global__ void k_genome_ranges(const uint64_t *__restrict__ poskey, const uint32_t *__restrict__ d_n, uint32_t cap,
                                const uint64_t *__restrict__ genome_off, uint64_t n_genomes, uint32_t *__restrict__ gs) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g > n_genomes) return;
    const uint32_t N = min(*d_n, cap);
    gs[g] = g == n_genomes ? N : (uint32_t)lower_bound_u64(poskey, N, genome_off[g] << 32);
}

// ---- duplicates (src/sketch.rs:594-600,605: a hash seen twice in one genome drops all its occurrences) ----
// One open-addressing table of survivor indices for the whole batch in global memory: genome g owns the slots
// [2 * gs[g], 2 * gs[g+1]) — load factor 1/2 whatever the genome's size or its share of repeats, so there is no
// table-overflow case.  Slots are only ever filled, and all occurrences of a hash walk the same probe sequence, so
// they all stop at the same slot: the first one that holds an occurrence of the hash.  The occurrence that fills
// it stays undecided unless another one arrives; every later occurrence drops itself and the one in the slot.
// No hash value or bit is reserved, so the rule holds for every c >= 1 (at c = 1 hashes use all 64 bits).
constexpr uint32_t DUP_EMPTY = 0xFFFFFFFFu;  // no survivor index (N <= 2^32 - 2)

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

// 32 hash bits scaled to [0, size): hashes are uniform below the threshold, so are these bits.  64-bit, so that a
// genome may own more than 2^32 slots.
__device__ __forceinline__ uint64_t dup_slot(uint64_t h, uint64_t size) { return __umul64hi((h >> 6) << 32, size); }

// flag[] = 3 (undecided) on entry; a hash occurring >= 2x in its genome leaves all its occurrences at 0 (dropped)
__global__ void __launch_bounds__(256)
k_dups(const uint64_t *__restrict__ hash, const uint32_t *__restrict__ gs, uint64_t n_genomes, uint32_t *__restrict__ table,
       uint8_t *__restrict__ flag) {
    __shared__ uint32_t s_lo, s_hi;
    const uint64_t N = gs[n_genomes], first = (uint64_t)blockIdx.x * 256;
    if (first >= N) return;
    const uint64_t i = first + threadIdx.x;
    const uint32_t g = dup_genome_of(gs, n_genomes, (uint32_t)min(i, N - 1), (uint32_t)first, (uint32_t)min(first + 255, N - 1),
                                     &s_lo, &s_hi);
    if (i >= N) return;
    const uint64_t size = 2ull * (gs[g + 1] - gs[g]);
    uint32_t *T = table + 2ull * gs[g];
    const uint64_t h = hash[i];
    for (uint64_t sl = dup_slot(h, size);;) {
        const uint32_t j = atomicCAS(&T[sl], DUP_EMPTY, (uint32_t)i);
        if (j == DUP_EMPTY) return;
        if (hash[j] == h) { flag[i] = 0; flag[j] = 0; return; }
        if (++sl == size) sl = 0;
    }
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

// poskey[i] = contig << 32 | pos and hash[i], i < N, in (contig, pos) order; N = *d_n (device memory), 1 <= cap < 2^32 - 1
// bounds the arrays.  The element-wise grids are sized for cap (threads past N return).  Returns SYL_ERR_UNSUPPORTED with
// the handle left empty when N > cap or *d_overflow (the slotted front half's slot overflow) is set: the caller redoes the
// batch on the sorted front half.  kt, the post-pass timer the front half started, stops before the host synchronisation.
static int genomes_back_half(syl_ctx *ctx, KernelTimer &kt, const uint64_t *poskey, const uint64_t *hash, const uint32_t *d_n,
                             uint64_t cap, const uint32_t *d_overflow, const uint64_t *d_contig_off, const uint64_t *d_genome_off,
                             uint64_t n_genomes, uint64_t min_spacing, int pseudotax, syl_genomes *out) {
    cudaStream_t st = ctx->stream;
    DevBuf<uint32_t> gs, dup_table, bk, bt, bk_off, bt_off, scan_k, scan_t, t1, t2, t3, t4;
    DevBuf<uint64_t> tmp_k, tmp_t;
    DevBuf<uint8_t> flag;
    SYL_TRY(gs.alloc(n_genomes + 1, st));
    k_genome_ranges<<<nblk(n_genomes + 1, 256), 256, 0, st>>>(poskey, d_n, (uint32_t)cap, d_genome_off, n_genomes, gs.p);
    const uint32_t *d_nc = gs.p + n_genomes;  // min(N, cap)
    SYL_TRY(flag.alloc(cap, st)); SYL_TRY(dup_table.alloc(2 * cap, st));
    SYL_CUDA(cudaMemsetAsync(flag.p, 3, cap, st));
    SYL_CUDA(cudaMemsetAsync(dup_table.p, 0xFF, 2 * cap * sizeof(uint32_t), st));
    k_dups<<<nblk(cap, 256), 256, 0, st>>>(hash, gs.p, n_genomes, dup_table.p, flag.p);
    k_spacing<<<nblk(cap, 256), 256, 0, st>>>(poskey, cap, min_spacing, flag.p, d_nc);
    const uint64_t nb = (cap + 1023) / 1024;
    SYL_TRY(bk.alloc(nb, st)); SYL_TRY(bt.alloc(nb, st)); SYL_TRY(bk_off.alloc(nb + 1, st)); SYL_TRY(bt_off.alloc(nb + 1, st));
    SYL_TRY(scan_k.alloc(cap, st)); SYL_TRY(scan_t.alloc(cap, st)); SYL_TRY(tmp_k.alloc(cap, st)); SYL_TRY(tmp_t.alloc(cap, st));
    k_flag_counts<<<(unsigned)nb, 256, 0, st>>>(flag.p, d_nc, bk.p, bt.p);
    SYL_TRY(scan_u32(ctx, bk.p, nb, bk_off.p, t1, t2));
    SYL_TRY(scan_u32(ctx, bt.p, nb, bt_off.p, t3, t4));
    k_scatter_flagged_blocks<<<(unsigned)nb, 1024, 0, st>>>(hash, flag.p, d_nc, bk_off.p, bt_off.p, tmp_k.p, pseudotax ? tmp_t.p : nullptr,
                                                            scan_k.p, scan_t.p);
    ctx->launches += 5;
    // per-genome offsets go straight into the handle; the k-mer arrays need the totals first
    out->has_tracked = pseudotax ? 1 : 0;
    out->stream = st;
    out->owner = tl_ctx;
    out->n = n_genomes;
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->kmer_off, (n_genomes + 1) * 8));
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->tracked_off, (n_genomes + 1) * 8));
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->gn_size, std::max<uint64_t>(n_genomes, 1) * 8));
    k_genome_offsets32<<<nblk(n_genomes + 1, 128), 128, 0, st>>>(gs.p, d_nc, d_genome_off, n_genomes, scan_k.p, scan_t.p, bk_off.p + nb,
                                                                 bt_off.p + nb, pseudotax, d_contig_off, out->kmer_off, out->tracked_off,
                                                                 out->gn_size);
    ctx->launches++;
    kt.stop();
    SYL_CUDA(cudaGetLastError());
    uint32_t *h32 = reinterpret_cast<uint32_t *>(ctx->h_counters + 4);  // N, kept, tracked, slot overflow
    SYL_CUDA(cudaMemcpyAsync(h32, d_n, 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpyAsync(h32 + 1, bk_off.p + nb, 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaMemcpyAsync(h32 + 2, bt_off.p + nb, 4, cudaMemcpyDeviceToHost, st));
    if (d_overflow) SYL_CUDA(cudaMemcpyAsync(h32 + 3, d_overflow, 4, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));  // the one synchronisation of the back half
    if (h32[0] > cap || (d_overflow && h32[3])) {
        hblock_free(out->owner, out->kmer_off); hblock_free(out->owner, out->tracked_off); hblock_free(out->owner, out->gn_size);
        out->kmer_off = out->tracked_off = out->gn_size = nullptr;
        return SYL_ERR_UNSUPPORTED;
    }
    const uint64_t total_kept = h32[1], total_tracked = pseudotax ? h32[2] : 0;
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->kmers, std::max<uint64_t>(total_kept, 1) * 8));
    SYL_TRY(hblock_alloc(out->owner, (void **)&out->tracked, std::max<uint64_t>(total_tracked, 1) * 8));
    out->total_kmers = total_kept;
    out->total_tracked = total_tracked;
    if (total_kept) SYL_CUDA(cudaMemcpyAsync(out->kmers, tmp_k.p, total_kept * 8, cudaMemcpyDeviceToDevice, st));
    if (total_tracked) SYL_CUDA(cudaMemcpyAsync(out->tracked, tmp_t.p, total_tracked * 8, cudaMemcpyDeviceToDevice, st));
    return SYL_OK;
}

// Slotted front half: k_seed writes every tile's survivors into the tile's own slot (SlotOut) in position order (its
// flush ranks the <= 512 survivors of a tile by window start); a scan of the per-tile counts and k_tile_compact make
// them one array.  No host synchronisation before the back half.  Exactly one of d_bases (ASCII) / d_packed (2-bit
// words) is set, here and in the functions below.
static int genomes_slotted(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases,
                           const uint64_t *d_contig_off, uint64_t n_contigs, const uint64_t *d_genome_off, uint64_t n_genomes,
                           int k, uint64_t c, uint64_t min_spacing, int pseudotax, int sem, syl_genomes *out) {
    cudaStream_t st = ctx->stream;
    const uint64_t n_tiles = seed_cta_tiles(n_bases);
    if (n_tiles * GEN_SLOT >= 0xFFFFFFFFull) { set_error("genome batch too large; split the batch"); return SYL_ERR_ARG; }
    const uint64_t cap = std::min<uint64_t>(n_tiles * GEN_SLOT, n_bases / c + n_bases / (4 * c) + 65536);  // compact survivors
    DevBuf<syl_survivor> slots;
    DevBuf<uint32_t> tile_cnt, toff, overflow, t1, t2;
    DevBuf<uint64_t> poskey, hash;
    SYL_TRY(slots.alloc(n_tiles * GEN_SLOT, st));
    SYL_TRY(tile_cnt.alloc(n_tiles, st)); SYL_TRY(toff.alloc(n_tiles + 1, st));
    SYL_TRY(overflow.alloc(1, st));
    SYL_CUDA(cudaMemsetAsync(overflow.p, 0, 4, st));
    SYL_CUDA(cudaMemsetAsync(ctx->d_counters, 0, 2 * sizeof(uint64_t), st));
    SeedJob job;
    job.d_bases = d_bases; job.d_packed = d_packed; job.n_bases = n_bases; job.d_rec_off = d_contig_off; job.off_bias = 0; job.n_rec = n_contigs;
    job.k = k; job.c = c; job.sem = sem; job.with_pos = 1; job.d_out = slots.p; job.cap = n_tiles * GEN_SLOT;
    job.d_count = reinterpret_cast<unsigned long long *>(ctx->d_counters);
    job.slot_cap = GEN_SLOT; job.d_tile_cnt = tile_cnt.p; job.d_slot_overflow = overflow.p;
    SYL_TRY(seed_enqueue(ctx, job));
    KernelTimer kt_post(ctx, SYL_KERNEL_GENOME_POST);
    SYL_TRY(scan_u32(ctx, tile_cnt.p, n_tiles, toff.p, t1, t2));   // toff[n_tiles] = N (device)
    SYL_TRY(poskey.alloc(cap, st)); SYL_TRY(hash.alloc(cap, st));
    k_tile_compact<<<nblk(n_tiles, 8), 256, 0, st>>>(slots.p, tile_cnt.p, toff.p, n_tiles, (uint32_t)cap, poskey.p, hash.p);
    ctx->launches++;
    return genomes_back_half(ctx, kt_post, poskey.p, hash.p, toff.p + n_tiles, cap, overflow.p, d_contig_off, d_genome_off,
                             n_genomes, min_spacing, pseudotax, out);
}

// Sorted front half, for every input: survivors with positions from seed_device (one host synchronisation, which
// also sizes the buffers), then one radix sort by (contig, pos) carrying the hash.
static int genomes_sorted(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases,
                          const uint64_t *d_contig_off, uint64_t n_contigs, const uint64_t *d_genome_off, uint64_t n_genomes,
                          int k, uint64_t c, uint64_t min_spacing, int pseudotax, int sem, syl_genomes *out) {
    cudaStream_t st = ctx->stream;
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
    KernelTimer kt_post(ctx, SYL_KERNEL_GENOME_POST);
    const uint64_t NA = std::max<uint64_t>(N, 1);
    DevBuf<uint64_t> key_b, hash_b;
    SYL_TRY(key_b.alloc(NA, st)); SYL_TRY(hash_b.alloc(NA, st));
    if (N) {
        DevBuf<uint64_t> key_a, hash_a;
        DevBuf<uint8_t> tmp;
        SYL_TRY(key_a.alloc(N, st)); SYL_TRY(hash_a.alloc(N, st));
        k_split<<<nblk(N, 256), 256, 0, st>>>(sv.p, N, key_a.p, hash_a.p);
        const int pos_bits = 32 + bits_for(n_contigs);
        size_t tb = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tb, key_a.p, key_b.p, hash_a.p, hash_b.p, N, 0, pos_bits, st);
        SYL_TRY(tmp.alloc(tb, st));
        SYL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, key_a.p, key_b.p, hash_a.p, hash_b.p, N, 0, pos_bits, st));
        ctx->launches += 2;
    }
    sv.release();
    // seed_device left N (< 2^32 - 1) in the u64 d_counters[0]: its low word is the back half's count
    return genomes_back_half(ctx, kt_post, key_b.p, hash_b.p, reinterpret_cast<const uint32_t *>(ctx->d_counters), NA, nullptr,
                             d_contig_off, d_genome_off, n_genomes, min_spacing, pseudotax, out);
}

int sketch_genomes_device(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases,
                          const uint64_t *d_contig_off, uint64_t n_contigs, const uint64_t *d_genome_off, uint64_t n_genomes,
                          int k, uint64_t c, uint64_t min_spacing, int pseudotax, int sem, syl_genomes *out) {
    const char *e = getenv("SYL_GENOME_POSTPASS");  // "sort" forces the sorted front half (tests); read per call
    const bool force_sort = e && std::string(e) == "sort";
    // slots hold 512 survivors per 32K-base tile: c >= 96 keeps the expected number below 350
    if (!force_sort && c >= 96 && n_bases && n_contigs && n_genomes) {
        const int rc = genomes_slotted(ctx, d_bases, d_packed, n_bases, d_contig_off, n_contigs, d_genome_off, n_genomes, k, c,
                                       min_spacing, pseudotax, sem, out);
        if (rc != SYL_ERR_UNSUPPORTED) return rc;
        // a slot or the compact arrays overflowed (low-complexity sequence): redo the batch on the sorted front half
    }
    return genomes_sorted(ctx, d_bases, d_packed, n_bases, d_contig_off, n_contigs, d_genome_off, n_genomes, k, c, min_spacing,
                          pseudotax, sem, out);
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
    Staged<uint8_t> sb;  // host memory: staged copies, alive until the call's last sync
    Staged<uint32_t> sp;
    Staged<uint64_t> sc, sg;
    if (packed) SYL_TRY(sp.init(ctx, mem, packed, (n_bases + 15) / 16));
    else SYL_TRY(sb.init(ctx, mem, bases, n_bases));
    SYL_TRY(sc.init(ctx, mem, contig_off, n_contigs + 1));
    if (individual) {  // every record is its own genome (src/sketch.rs:481-548)
        n_genomes = n_contigs;
        SYL_TRY(sg.buf.alloc(n_contigs + 1, st));
        k_iota64<<<nblk(n_contigs + 1, 256), 256, 0, st>>>(sg.buf.p, n_contigs + 1);
        ctx->launches++;
        sg.p = sg.buf.p;
    } else {
        SYL_TRY(sg.init(ctx, mem, genome_off, n_genomes + 1));
    }
    syl_genomes *g = new (std::nothrow) syl_genomes();
    if (!g) return SYL_ERR_OOM;
    g->device = ctx->device;
    g->k = k;
    g->c = c;
    int rc = sketch_genomes_device(ctx, sb.p, sp.p, n_bases, sc.p, n_contigs, sg.p, n_genomes, k, c, min_spacing,
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
    // tracked_off says whether the sketches carry tracked k-mers; tracked may be NULL when there are none (an empty
    // torch tensor has no address)
    if (nt && !tracked) { set_error("tracked_off counts tracked k-mers but tracked is NULL"); return SYL_ERR_ARG; }
    syl_genomes *g = new (std::nothrow) syl_genomes();
    if (!g) return SYL_ERR_OOM;
    g->device = ctx->device; g->k = k; g->c = c;
    g->has_tracked = tracked_off ? 1 : 0;
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
