// seed.cu — FracMinHash seeding on sm_90a.
//
// Replaces, for a whole batch of records at once, the reference's per-record
//   extract_markers            (src/sketch.rs:53-69  -> src/avx2_seeding.rs:33-148 / src/seeding.rs:86-146)
//   extract_markers_positions  (src/sketch.rs:71-93  -> src/avx2_seeding.rs:151-266 / src/seeding.rs:148-209)
//
// Formulation (nothing here mirrors the AVX2 traversal; only its window *set* is kept):
//   * the batch is one flat buffer, ASCII or 2-bit packed; a CTA owns a tile of SEED_TILE window-start
//     positions (seed_kernel.cuh, k_seed)
//   * the tile (+halo) is staged HBM -> shared memory with one TMA bulk copy (cp.async.bulk +
//     mbarrier complete_tx), then packed ONCE into two 2-bit streams (2-bit input: the forward
//     stream is the staged words):
//        fw: forward codes, MSB-first     -> forward k-mer of any window = one 64-bit funnel extract
//        cw: complement codes, LSB-first  -> reverse-complement k-mer  = one 64-bit funnel extract
//     so windows are independent (no serial roll, no per-window byte loads)
//   * the records overlapping the tile are cut into runs of <= W (24, 30 or 32) consecutive VALID window
//     starts (the AVX2 lane rule is just "start < 4*((L-k+1)/4)"), one run per thread, so no
//     issue slots are spent on windows that straddle a record boundary (20 % of all windows
//     for 150 bp reads)
//   * per window: 2+2 funnel shifts, 64-bit min, the 64-bit hash (4 IMAD-pipe multiplies +
//     3 ALU-pipe xor-shifts), one compare of the high word against the threshold
//   * survivors (1/c of windows) are staged in shared memory and flushed with one global
//     atomic per CTA
#include <algorithm>
#include <cstdlib>

#include "seed_kernel.cuh"

namespace syl {

// tile t -> index of the record that contains flat position t*tile
__global__ void k_tile_first_rec(const uint64_t *__restrict__ rec_off, uint64_t off_bias, uint64_t n_rec,
                                 uint64_t n_tiles, uint64_t tile, uint32_t *__restrict__ tile_rec) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > n_tiles) return;
    if (t == n_tiles) {
        tile_rec[t] = (uint32_t)(n_rec - 1);
        return;
    }
    uint64_t pos = t * tile + off_bias;
    // upper_bound over rec_off[0..n_rec]: first i with rec_off[i] > pos
    uint64_t lo = 0, hi = n_rec + 1;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (rec_off[mid] > pos) hi = mid; else lo = mid + 1;
    }
    uint64_t r = lo == 0 ? 0 : lo - 1;
    if (r >= n_rec) r = n_rec - 1;
    tile_rec[t] = (uint32_t)r;
}

// cost of a record with w windows at run length W: ceil(w / W) runs, each W windows plus ~1.5
// windows' worth of set-up (stream realignment, table look-ups)
static int pick_run_length(uint64_t mean_len, int k, int sem, int with_pos) {
    static const int forced = []() { const char *e = getenv("SYL_SEED_W"); return e ? atoi(e) : 0; }();
    static const int opts[] = {32, 30, 24};
    if (forced) { for (int w : opts) if (w == forced) return w; }
    const uint64_t w = valid_windows(mean_len, (uint32_t)k, sem, with_pos);
    if (w == 0 || w > 4096) return SEED_W_MAX;
    int best = SEED_W_MAX;
    double best_cost = 1e300;
    for (int W : opts) {
        const double cost = (double)((w + W - 1) / W) * (W + 1.5);
        if (cost < best_cost - 1e-9) { best_cost = cost; best = W; }
    }
    return best;
}

// Measured on 1 Gbp of 150 bp reads (one H100 SXM, 400 W): k_seed 1.6-1.9 ms; the hot loop alone
// (scripts/hotloop_bench.cu) sustains 0.66 T windows/s = 1.22 ms for the same windows, so the phases around
// the loop cost about 0.4-0.5 ms of the kernel.
uint64_t seed_cta_tiles(uint64_t n_bases) { return (n_bases + SEED_TILE - 1) / SEED_TILE; }
uint64_t seed_cta_tile_bases() { return SEED_TILE; }

// Enqueue the seeding of one batch on the ctx stream.  No host synchronisation and no counter reset:
// survivors / events are appended to job.d_out at the running device counter job.d_count[0] (entries
// past job.cap are counted but dropped; the caller compares the final count with cap), pending
// event indices at job.d_count[1].
int seed_enqueue(syl_ctx *ctx, const SeedJob &job) {
    if (job.emit_events && (!job.d_pend || job.cap >= 0xFFFFFFFFull)) { set_error("event emission needs a pending list and cap < 2^32"); return SYL_ERR_ARG; }
    if (job.c == 0) { set_error("c must be >= 1"); return SYL_ERR_ARG; }
    if (!(job.k == 21 || job.k == 31)) {
        set_error("k must be 21 or 31 (the reference panics otherwise, src/avx2_seeding.rs:46-52)");
        return SYL_ERR_UNSUPPORTED;
    }
    if (job.sem != SYL_SEM_SCALAR && job.sem != SYL_SEM_AVX2) { set_error("bad sem"); return SYL_ERR_ARG; }
    if (job.n_rec == 0 || job.n_bases == 0) return SYL_OK;
    if (job.n_rec >= 0xFFFFFFFFull) { set_error("more than 2^32-2 records in one batch"); return SYL_ERR_ARG; }
    const void *in = job.d_packed ? (const void *)job.d_packed : (const void *)job.d_bases;
    if ((reinterpret_cast<uintptr_t>(in) & 15u) != 0) {
        set_error("device base buffer must be 16-byte aligned (TMA bulk copy)");
        return SYL_ERR_ARG;
    }
    const bool packed = job.d_packed != nullptr;
    cudaStream_t st = ctx->stream;
    // Run length: every record is cut into runs of W windows and a thread always pays for a full
    // run, so for fixed-length reads W should divide the per-read window count (150 bp, k=31:
    // 120 windows = 4 x 30).  Chosen from the mean record length; long records get 32.
    const int W = pick_run_length(job.n_bases / job.n_rec, job.k, job.sem, job.with_pos);
    const uint64_t n_tiles = seed_cta_tiles(job.n_bases);
    DevBuf<uint32_t> tile_rec;
    SYL_TRY(tile_rec.alloc(n_tiles + 1, st));
    {
        const int bs = 256;
        const uint64_t nb = (n_tiles + 1 + bs - 1) / bs;
        k_tile_first_rec<<<(unsigned)nb, bs, 0, st>>>(job.d_rec_off, job.off_bias, job.n_rec, n_tiles, SEED_TILE, tile_rec.p);
        ctx->launches++;
    }
    // events of one part of a sample (sample_parts.hpp): hashes below the part's upper bound hi <= fmh_threshold
    const uint64_t thr = job.emit_events ? std::min(job.hi, fmh_threshold(job.c)) : fmh_threshold(job.c);
    const ImadConst ic = {{0u, 0u, 0u}, 1u, 0u};
    const GroupOut go{job.emit_events ? job.d_group_cnt : nullptr, job.Mb, job.nbk, job.ng, job.slot, job.g0, job.lo};
    const SlotOut slot{job.emit_events ? 0u : job.slot_cap, job.d_tile_cnt, job.d_slot_overflow};
    const size_t smem = sizeof(SeedSmem);
    const seed_kern_t kern = job.emit_events ? (job.k == 31 ? seed_kernels_k31_ev(W, packed) : seed_kernels_k21_ev(W, packed))
                                             : (job.k == 31 ? seed_kernels_k31_sv(W, packed) : seed_kernels_k21_sv(W, packed));
    SYL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    KernelTimer kt(ctx, SYL_KERNEL_SEED);
    kern<<<(unsigned)n_tiles, SEED_THREADS, smem, st>>>(
        reinterpret_cast<const uint8_t *>(in), job.n_bases, job.d_rec_off, job.off_bias, tile_rec.p, thr, job.sem, job.with_pos,
        job.d_out, slot.cap ? 0 : job.cap, job.d_count, ic, job.rec_base, job.no_dedup, job.d_pend, go, slot);
    kt.stop();
    if (ctx->timing) ctx->seed_bases += job.n_bases;
    ctx->launches++;
    SYL_CUDA(cudaGetLastError());
    return SYL_OK;
}

// Synchronous form: device-resident inputs, survivors to a device buffer. *n_out is the true
// number of survivors even when it exceeds cap (then SYL_ERR_CAPACITY).
// d_rec_off[i] - off_bias is the start of record i inside the batch (off_bias lets a caller pass a
// slice of a larger offset array unchanged).  Exactly one of d_bases (ASCII) / d_packed (2-bit words) is set.
int seed_device(syl_ctx *ctx, const uint8_t *d_bases, const uint32_t *d_packed, uint64_t n_bases, const uint64_t *d_rec_off,
                uint64_t off_bias, uint64_t n_rec, int k, uint64_t c, int sem, int with_pos, syl_survivor *d_out,
                uint64_t cap, uint64_t *n_out) {
    *n_out = 0;
    cudaStream_t st = ctx->stream;
    SeedJob job;
    job.d_bases = d_bases; job.d_packed = d_packed; job.n_bases = n_bases; job.d_rec_off = d_rec_off; job.off_bias = off_bias; job.n_rec = n_rec;
    job.k = k; job.c = c; job.sem = sem; job.with_pos = with_pos; job.d_out = d_out; job.cap = cap;
    job.d_count = reinterpret_cast<unsigned long long *>(ctx->d_counters);
    SYL_CUDA(cudaMemsetAsync(ctx->d_counters, 0, 2 * sizeof(uint64_t), st));  // CNT_EVENTS, CNT_PENDING
    SYL_TRY(seed_enqueue(ctx, job));
    SYL_CUDA(cudaMemcpyAsync(ctx->h_counters + CNT_EVENTS, ctx->d_counters + CNT_EVENTS, 8, cudaMemcpyDeviceToHost, st));
    SYL_CUDA(cudaStreamSynchronize(st));
    *n_out = ctx->h_counters[CNT_EVENTS];
    if (*n_out > cap) {
        set_error("survivor buffer too small");
        return SYL_ERR_CAPACITY;
    }
    return SYL_OK;
}

}  // namespace syl
