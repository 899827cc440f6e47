// contain_calls.cu — the query / profile calls: argument checks, the samples of a call batch by batch (device handles
// or host arrays), sharded databases (syl_db_shards) swept shard by shard, and one driver that every call ends in.
#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <functional>
#include <new>
#include <vector>

#include "contain.hpp"
#include "ingest.hpp"
#include "sample_batches.hpp"
#include "scan_plan.hpp"
#include "shard_cut.hpp"

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
int check_contain_args(syl_ctx *ctx, int k, uint64_t c, bool has_tracked, bool profile, const syl_sample *const *samples,
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
int copy_rows(const std::vector<syl_ani_row> &out, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    *n_rows = out.size();
    if (out.size() > cap) { set_error("row buffer too small"); return SYL_ERR_CAPACITY; }
    std::copy(out.begin(), out.end(), rows);
    return SYL_OK;
}

__global__ void k_sum_counts(const uint32_t *__restrict__ count, uint64_t n, unsigned long long *__restrict__ out) {
    unsigned long long acc = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) acc += count[i];
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

// Device handles as the views the joins take, and what -u needs to know of them (the sum of the counts is computed on the
// device once per handle, and only for -u).
int handle_views(syl_ctx *ctx, const syl_sample *const *samples, uint32_t n, bool unknown, std::vector<SampleView> &views,
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
    bool scan = false;              // pass 1 of a shards call by the scan formulation (decided at the call's entry)
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

// Device handles (handle_views): batches of at most max_pairs pairs.
struct HandleSamples : SampleSource {
    std::vector<SampleView> all;
    uint64_t max_pairs;
    explicit HandleSamples(uint64_t mp) : max_pairs(mp) {}
    void batches(uint64_t G, std::vector<uint32_t> &first) const override {
        const uint32_t S = (uint32_t)all.size();
        const uint32_t per = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(S, max_pairs / std::max<uint64_t>(G, 1)));
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
// batch (hash, count and rebased offsets), filled on the ctx's copy stream and sorted there by hash within each sample
// (one segmented sort per batch, into the slot or the shared second buffer, whichever it ends in), while the ctx stream
// joins the other slot.  A SlotHandoff orders the two streams; the host waits only where the joins already do.
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
    } slot[2];
    DevBuf<uint64_t> alt_hash;
    DevBuf<uint32_t> alt_count;
    DevBuf<uint8_t> tmp;
    SlotHandoff<2> handoff;  // after the buffers it orders (ingest.hpp)
    int cur = -1;  // slot of the last views()

    HostSamples(syl_ctx *c, const syl_host_samples *s) : ctx(c), in(s) {}
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
        cudaStream_t cs = nullptr, st = ctx->stream;
        SYL_TRY(ingest_copy_stream(ctx, &cs));
        SYL_TRY(handoff.init(cs, st));
        for (Slot &sl : slot) {
            SYL_TRY(sl.hash.alloc(kmers, st)); SYL_TRY(sl.count.alloc(kmers, st)); SYL_TRY(sl.off.alloc(S + 1, st));
        }
        SYL_TRY(alt_hash.alloc(kmers, st)); SYL_TRY(alt_count.alloc(kmers, st)); SYL_TRY(tmp.alloc(tb, st));
        return handoff.fence();
    }
    // samples [s0, s1) into slot k, once the joins of its last batch are done
    int stage(int k, uint32_t s0, uint32_t s1) {
        if (!handoff.cs) SYL_TRY(init());
        Slot &sl = slot[k];
        SYL_TRY(handoff.before_copy(k));
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
            SYL_CUDA(cub::DeviceSegmentedSort::SortPairs(tmp.p, tb, dk, dv, (int)n, (int)(s1 - s0), sl.off.p, sl.off.p + 1, handoff.cs));
            ctx->launches += 4;
            if (dk.selector) sl.hash.swap(alt_hash);
            if (dv.selector) sl.count.swap(alt_count);
        }
        SYL_TRY(handoff.copied_in(k));
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
        SYL_TRY(handoff.take(k));
        v.resize(s1 - s0);
        for (uint32_t i = s0; i < s1; i++) {
            const uint64_t o = sl.h_off[i - sl.s0];
            v[i - s0] = {sl.hash.p + o, sl.count.p + o, sl.h_off[i + 1 - sl.s0] - o};
        }
        cur = k;
        return SYL_OK;
    }
    void done() override {
        if (cur >= 0) handoff.done(cur);
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

// Whether a call of this shape scans (scan_plan.hpp), with SYL_DB_SCAN (read per call) forcing either path where the
// samples fit one batch
static bool plan_scan(const ScanShape &shape) { return scan_decision(shape, scan_forced(getenv("SYL_DB_SCAN"))); }

// Genomes of one scan chunk at most: a chunk's joins hold at most PAIRS_PER_CALL (sample, genome) pairs
static uint64_t scan_chunk_genomes(uint32_t S) { return std::max<uint64_t>(PAIRS_PER_CALL / std::max<uint32_t>(S, 1), 1); }

static uint64_t scan_chunk_env() {  // SYL_DB_SCAN_CHUNK: genome k-mers per scan chunk (tests; read per call)
    if (const char *e = getenv("SYL_DB_SCAN_CHUNK")) {
        const long long v = atoll(e);
        if (v >= 1) return (uint64_t)v;
    }
    return SCAN_CHUNK;
}

// Pass 1 (syl_query) of all samples of src (one batch) by the scan formulation: the genome k-mers cross the link chunk by
// chunk (whole genomes) on the ctx's copy stream into two device buffers, chunk i + 1 while chunk i is scanned, and
// each chunk is a query of its genomes (contain_fast with the chunk).  rows: by chunk, then by (sample, genome);
// row.genome is the global index.  Its blocks go back to the ctx cache when it returns.  src holds all samples in one
// batch (scan_one_batch).
static int scan_sweep(syl_db_shards *s, SampleSource &src, const syl_contain_params *p, std::vector<syl_ani_row> &rows) {
    syl_ctx *ctx = s->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t S = (uint32_t)src.metas.size();
    SYL_TRY(cache_trim(ctx));
    const auto t0 = std::chrono::steady_clock::now();
    // kernel milliseconds of SYL_DEBUG_TIMING's line (with syl_ctx_enable_timing; else they stay 0)
    double scan0 = 0., stats0 = 0., scan1 = 0., stats1 = 0.;
    if (debug_timing()) {
        SYL_TRY(syl_ctx_kernel_time(ctx, SYL_KERNEL_SCAN, &scan0, nullptr, 0));
        SYL_TRY(syl_ctx_kernel_time(ctx, SYL_KERNEL_STATS, &stats0, nullptr, 0));
    }
    const uint64_t h2d0 = ctx->ingest_h2d_bytes;
    std::vector<SampleView> v;
    SYL_TRY(src.views(0, S, v));
    DevBuf<SampleTable> tables;
    DevBuf<uint32_t> dir, fp;
    std::vector<SampleTable> ht;
    SYL_TRY(build_tables(ctx, v.data(), S, tables, dir, fp, ht));
    std::vector<uint64_t> first;
    cut_scan_chunks(s->kmer_off, s->G, scan_chunk_env(), scan_chunk_genomes(S), first);
    const size_t nc = first.size() - 1;
    uint64_t max_n = 0, max_g = 0;
    for (size_t i = 0; i < nc; i++) {
        max_n = std::max(max_n, s->kmer_off[first[i + 1]] - s->kmer_off[first[i]]);
        max_g = std::max(max_g, first[i + 1] - first[i]);
    }
    struct Slot { DevBuf<uint64_t> kmers, off; DevBuf<uint32_t> glen; } slot[2];
    SlotHandoff<2> handoff;  // after the slots (ingest.hpp)
    cudaStream_t cs = nullptr;
    SYL_TRY(ingest_copy_stream(ctx, &cs));
    for (Slot &sl : slot) {
        SYL_TRY(sl.kmers.alloc(max_n, st));
        SYL_TRY(sl.off.alloc(max_g + 1, st));
        SYL_TRY(sl.glen.alloc(max_g, st));
    }
    SYL_TRY(handoff.init(cs, st));
    SYL_TRY(handoff.fence());  // cached blocks: earlier work
    const bool pinned = s->kmers && ptr_kind(s->kmers) == PtrKind::PINNED;
    std::vector<uint64_t> h_off;
    std::vector<uint32_t> h_glen;
    // chunk i into slot i % 2 on the copy stream, once the scan of the chunk before it in that slot is done
    auto stage = [&](size_t i) -> int {
        Slot &sl = slot[i % 2];
        const uint64_t a = first[i], G = first[i + 1] - a, k0 = s->kmer_off[a];
        SYL_TRY(handoff.before_copy(i % 2));
        h_off.resize(G + 1);
        h_glen.resize(G);
        for (uint64_t g = 0; g <= G; g++) h_off[g] = s->kmer_off[a + g] - k0;
        for (uint64_t g = 0; g < G; g++) h_glen[g] = (uint32_t)(h_off[g + 1] - h_off[g]);
        SYL_TRY(ingest_copy(ctx, sl.off.p, h_off.data(), (G + 1) * 8, false));  // pageable: staged before it returns
        SYL_TRY(ingest_copy(ctx, sl.glen.p, h_glen.data(), G * 4, false));
        SYL_TRY(ingest_copy(ctx, sl.kmers.p, s->kmers + k0, h_off[G] * 8, pinned));
        return handoff.copied_in(i % 2);
    };
    if (nc) SYL_TRY(stage(0));
    for (size_t i = 0; i < nc; i++) {
        Slot &sl = slot[i % 2];
        SYL_TRY(handoff.take(i % 2));
        syl_db db;
        db.device = ctx->device;
        db.n_genomes = first[i + 1] - first[i];
        db.genome_base = (uint32_t)first[i];
        db.glen = sl.glen.p;
        db.k = s->k;
        db.c = s->c;
        db.has_tracked = s->tracked_off ? 1 : 0;
        const ScanChunk ch{sl.kmers.p, sl.off.p, s->kmer_off[first[i + 1]] - s->kmer_off[first[i]], tables.p};
        bool next_staged = i + 1 >= nc;
        std::function<int()> next;
        if (!next_staged) next = [&] { next_staged = true; return stage(i + 1); };
        std::vector<syl_ani_row> part;
        JoinRoom room = src.room;
        room.s0 = 0;
        SYL_TRY(contain_fast(ctx, &db, v.data(), src.metas.data(), S, p, false, part, next, &room, &ch));
        SYL_TRY(handoff.done(i % 2));
        if (!next_staged) SYL_TRY(stage(i + 1));
        rows.insert(rows.end(), part.begin(), part.end());
    }
    src.done();
    cudaStreamSynchronize(st);  // the handoff drains the copy stream as it returns
    if (debug_timing()) {
        SYL_TRY(syl_ctx_kernel_time(ctx, SYL_KERNEL_SCAN, &scan1, nullptr, 0));
        SYL_TRY(syl_ctx_kernel_time(ctx, SYL_KERNEL_STATS, &stats1, nullptr, 0));
        fprintf(stderr, "[db scan] samples %u chunks %zu genome k-mers %llu: H2D %llu bytes (%s), scan %.1f ms, stats %.1f ms, pass 1 %.1f ms\n",
                S, nc, (unsigned long long)s->kmer_off[s->G], (unsigned long long)(ctx->ingest_h2d_bytes - h2d0),
                pinned ? "pinned" : "pageable", scan1 - scan0, stats1 - stats0, ms_since(t0));
    }
    return SYL_OK;
}

static ScanShape shards_shape(const syl_db_shards *s, uint32_t S, uint64_t sample_kmers, bool one_batch) {
    const bool pinned = s->kmers && ptr_kind(s->kmers) == PtrKind::PINNED;
    return ScanShape{s->kmer_off[s->G], s->tracked_off ? s->tracked_off[s->G] : 0, s->G, S, sample_kmers, one_batch, pinned};
}

// Pass 1 (syl_query) of every sample of src against every shard in turn: each shard's index is built once, joined with
// all samples batch by batch, and freed before the next one is built; or, when the call scans (src.scan), scan_sweep.
// rows: by shard, then by (sample, genome); row.genome is the global index.
static int shards_sweep(syl_db_shards *s, SampleSource &src, const syl_contain_params *p, std::vector<syl_ani_row> &rows) {
    syl_ctx *ctx = s->ctx;
    if (src.scan) {
        SYL_TRY(scan_sweep(s, src, p, rows));
        return cache_trim(ctx);  // the scan's blocks are back in the cache once scan_sweep has returned
    }
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
        if (debug_timing())
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
    SYL_TRY(check_db_size(nk, nt, n));
    const DbInput in{SYL_MEM_HOST, {s->pinned, s->pinned + nk}, {ko.data(), to.data()}, n, {nk, nt}};
    syl_db *db = nullptr;
    SYL_TRY(db_build(s->ctx, in, gsz.data(), 1, s->k, s->c, 0, &db));
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
    if (debug_timing())
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

// Every query and profile call after its checks: the samples of src against the shards (shards_call), or against one
// index in the source's batches.  key: the samples of the call (shards_call).
static int contain_call(syl_ctx *ctx, const syl_db *db, syl_db_shards *sh, SampleSource &src, const std::vector<const void *> &key,
                        const syl_contain_params *p, bool profile, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (sh) return shards_call(sh, src, key, p, profile, rows, cap, n_rows);
    if (db->n_genomes == 0 || src.metas.empty()) return SYL_OK;  // *n_rows is 0 since the checks
    std::vector<uint32_t> first;
    src.batches(db->n_genomes, first);
    std::vector<syl_ani_row> out;
    SYL_TRY(join_batches(ctx, db, src, first, nullptr, p, profile, out));
    return copy_rows(out, rows, cap, n_rows);
}

// k-mer size, sketch parameter and whether there are tracked k-mers, of the database of a call (one index or shards)
struct DbParams { int k; uint64_t c; bool tracked; };
static DbParams db_params(const syl_db *db, const syl_db_shards *sh) {
    return db ? DbParams{db->k, db->c, db->has_tracked != 0} : DbParams{sh->k, sh->c, sh->tracked_off != nullptr};
}

// syl_query / syl_profile (db) and syl_query_shards / syl_profile_shards (sh)
static int handle_call(syl_ctx *ctx, const syl_db *db, syl_db_shards *sh, const syl_sample *const *samples, uint32_t n,
                       const syl_contain_params *p, bool profile, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!db && !sh) { set_error("NULL argument"); return SYL_ERR_ARG; }
    const DbParams d = db_params(db, sh);
    SYL_TRY(check_contain_args(ctx, d.k, d.c, d.tracked, profile, samples, n, p, rows, cap, n_rows));
    if (sh && ctx != sh->ctx) { set_error("db shards used with another ctx than the one that created them"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    HandleSamples src(db ? UINT64_MAX : PAIRS_PER_CALL);  // one index: all samples in one join (contain_fast sizes it)
    SYL_TRY(handle_views(ctx, samples, n, p->estimate_unknown != 0, src.all, src.metas));
    if (sh) {  // handles are resident already: the scan takes them all at once
        uint64_t kmers = 0;
        for (const SampleView &v : src.all) kmers += v.n;
        src.scan = plan_scan(shards_shape(sh, n, kmers, true));
    }
    return contain_call(ctx, db, sh, src, std::vector<const void *>(samples, samples + n), p, profile, rows, cap, n_rows);
}

// the device budget of host samples: syl_ctx_set_sample_memory's, or (0) free memory plus the ctx's cached free blocks
static int sample_budget(syl_ctx *ctx, uint64_t *budget) {
    *budget = ctx->sample_budget;
    if (!*budget) {
        size_t free_b = 0, total_b = 0;
        SYL_CUDA(cudaMemGetInfo(&free_b, &total_b));
        *budget = free_b;
        for (const auto &b : ctx->free_blocks) *budget += b.second;
    }
    return SYL_OK;
}

// What a batch of host samples costs (sample_batches.hpp), and SYL_SAMPLE_BATCH=N (read per call): at most N samples
// per batch (0: no cap)
constexpr BatchCost HOST_BATCH_COST{36, 4 * 8 + sizeof(SampleView) + 96 * ROW_BYTES, 16, COV_BINS * 4 + 16, 256 * ROW_BYTES + (1u << 20)};
static uint32_t sample_batch_env() { const char *e = getenv("SYL_SAMPLE_BATCH"); return e ? (uint32_t)std::max(0, atoi(e)) : 0; }

// the batches of host samples against G genomes per join, within `budget`
static BatchPlanResult plan_host_batches(const uint64_t *off, uint32_t S, uint64_t G, uint64_t budget, std::vector<uint32_t> &plan,
                                         uint32_t *bad, uint64_t *need) {
    return plan_sample_batches(off, S, G, budget, PAIRS_PER_CALL, 0x7FFFFFFFull, sample_batch_env(), HOST_BATCH_COST, plan, bad, need);
}

// Whether S host samples of `kmers` k-mers together, the largest n_max, fit the one batch a scan call stages them in:
// the batch cost of plan_host_batches against a scan chunk's genomes, plus the samples' tables (6 bytes per k-mer), within
// the sample budget less the two staging chunks; SYL_SAMPLE_BATCH=N below S says no.  The decision of the call and of
// syl_db_scan_plan.
static int scan_one_batch(syl_ctx *ctx, uint32_t S, uint64_t kmers, uint64_t n_max, bool *one) {
    uint64_t budget = 0;
    SYL_TRY(sample_budget(ctx, &budget));
    const uint64_t staging = 2 * (8 * scan_chunk_env() + 12 * scan_chunk_genomes(S)), tables = 6 * kmers + 256 * (uint64_t)S;
    const uint32_t forced = sample_batch_env();
    const unsigned __int128 bytes = (unsigned __int128)2 * batch_bytes(HOST_BATCH_COST, kmers, S, n_max, scan_chunk_genomes(S)) + staging + tables;
    *one = S && kmers <= 0x7FFFFFFFull && bytes <= budget && (!forced || S <= forced);
    return SYL_OK;
}

// syl_query_host_samples / syl_profile_host_samples
static int host_samples_call(syl_ctx *ctx, const syl_db *db, syl_db_shards *sh, const syl_host_samples *s,
                             const syl_contain_params *p, bool profile, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    if (!ctx || !s || !p || !n_rows || (cap && !rows)) { set_error("NULL argument"); return SYL_ERR_ARG; }
    if ((db != nullptr) == (sh != nullptr)) { set_error("exactly one of db and shards must be given"); return SYL_ERR_ARG; }
    *n_rows = 0;
    const uint32_t S = s->n_samples;
    if (!s->off || (S && (!s->c || !s->mean_read_length))) { set_error("NULL argument"); return SYL_ERR_ARG; }
    SYL_TRY(check_host_offsets(s->off, nullptr, S));
    if (s->off[S] && (!s->hash || !s->count)) { set_error("off counts k-mers but hash or count is NULL"); return SYL_ERR_ARG; }
    const DbParams d = db_params(db, sh);
    for (uint32_t i = 0; i < S; i++) SYL_TRY(check_sample_kc(d.k, d.c, s->k, s->c[i]));
    SYL_TRY(check_params(d.k, d.tracked, profile, p));
    if (sh && ctx != sh->ctx) { set_error("db shards used with another ctx than the one that created them"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    HostSamples src(ctx, s);
    for (int a = 0; a < 2 && s->off[S]; a++) {  // pinned arrays are copied as they are, pageable ones through the ring
        const PtrKind kind = ptr_kind(a ? (const void *)s->count : (const void *)s->hash);
        if (kind == PtrKind::DEVICE || kind == PtrKind::MANAGED) { set_error("host samples: a device pointer was given"); return SYL_ERR_ARG; }
        (a ? src.pinned_count : src.pinned_hash) = kind == PtrKind::PINNED;
    }
    // the plan: the device budget of syl_ctx_set_sample_memory (0: free memory once the ctx's staging ring exists, plus
    // the ctx's cached free blocks), less the largest shard's build (16 bytes per entry)
    cudaStream_t cs = nullptr;
    SYL_TRY(ingest_copy_stream(ctx, &cs));
    uint64_t budget = 0, index = 0;
    SYL_TRY(sample_budget(ctx, &budget));
    // the joins' allocations beyond the plan are held to the budget on top of the bytes the ctx holds in use now
    uint64_t live = ctx->cached_bytes + ctx->transient_bytes;
    for (const auto &b : ctx->free_blocks) live -= b.second;
    src.room.limit = live + budget;
    src.room.budget = budget;
    if (sh) {  // a scan stages all samples as one batch and builds no index
        uint64_t n_max = 0;
        for (uint32_t i = 0; i < S; i++) n_max = std::max<uint64_t>(n_max, s->off[i + 1] - s->off[i]);
        bool one = false;
        SYL_TRY(scan_one_batch(ctx, S, s->off[S], n_max, &one));
        src.scan = plan_scan(shards_shape(sh, S, s->off[S], one));
    }
    if (src.scan) {
        src.plan = {0, S};
        src.plan_G = scan_chunk_genomes(S);
    } else if (sh) {
        for (size_t i = 0; i + 1 < sh->first.size(); i++) {
            const uint64_t a = sh->first[i], b = sh->first[i + 1];
            src.plan_G = std::max(src.plan_G, b - a);
            index = std::max(index, 16 * (sh->kmer_off[b] - sh->kmer_off[a] + (sh->tracked_off ? sh->tracked_off[b] - sh->tracked_off[a] : 0)));
        }
    } else {
        src.plan_G = db->n_genomes;
    }
    uint32_t bad = 0;
    uint64_t need = 0;
    const BatchPlanResult pr = src.scan ? BATCH_OK
                                        : plan_host_batches(s->off, S, src.plan_G, budget > index ? budget - index : 0, src.plan, &bad, &need);
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
    const std::vector<const void *> key{s->hash, s->count, s->off, s->c, s->mean_read_length, (const void *)(uintptr_t)S};
    return contain_call(ctx, db, sh, src, key, p, profile, rows, cap, n_rows);
}

}  // namespace syl

using namespace syl;

extern "C" {

int syl_query(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
              const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return handle_call(ctx, db, nullptr, samples, n_samples, p, false, rows, cap, n_rows);
}

int syl_profile(syl_ctx *ctx, const syl_db *db, const syl_sample *const *samples, uint32_t n_samples,
                const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return handle_call(ctx, db, nullptr, samples, n_samples, p, true, rows, cap, n_rows);
}

int syl_db_shards_create(syl_ctx *ctx, const uint64_t *kmers, const uint64_t *kmer_off, const uint64_t *tracked,
                         const uint64_t *tracked_off, const uint64_t *gn_size, uint64_t n_genomes, int k, uint64_t c,
                         uint64_t max_entries, syl_db_shards **out) {
    if (!ctx || !kmer_off || !out) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *out = nullptr;
    if (n_genomes > 0xFFFFFFFFull) { set_error("more than 2^32 genomes: row.genome is 32 bits"); return SYL_ERR_ARG; }
    SYL_ENTER(ctx);
    for (const uint64_t *a : {kmers, kmer_off, tracked, tracked_off, gn_size})  // the sweep reads them on the host
        if (a && ptr_kind(a) == PtrKind::DEVICE) { set_error("db shards borrow host arrays; a device pointer was given"); return SYL_ERR_ARG; }
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
    return handle_call(ctx, nullptr, s, samples, n_samples, p, false, rows, cap, n_rows);
}

int syl_profile_shards(syl_ctx *ctx, syl_db_shards *s, const syl_sample *const *samples, uint32_t n_samples,
                       const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return handle_call(ctx, nullptr, s, samples, n_samples, p, true, rows, cap, n_rows);
}

int syl_query_host_samples(syl_ctx *ctx, const syl_db *db, syl_db_shards *shards, const syl_host_samples *s,
                           const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return host_samples_call(ctx, db, shards, s, p, false, rows, cap, n_rows);
}

int syl_profile_host_samples(syl_ctx *ctx, const syl_db *db, syl_db_shards *shards, const syl_host_samples *s,
                             const syl_contain_params *p, syl_ani_row *rows, uint64_t cap, uint64_t *n_rows) {
    return host_samples_call(ctx, db, shards, s, p, true, rows, cap, n_rows);
}

int syl_db_scan_plan(syl_ctx *ctx, uint64_t n_kmers, uint64_t n_tracked, uint64_t n_genomes, uint32_t n_samples,
                     uint64_t sample_kmers, int *scan) {
    if (!ctx || !scan) { set_error("NULL argument"); return SYL_ERR_ARG; }
    *scan = 0;
    SYL_ENTER(ctx);
    // one batch as the call decides it, for n_samples equal host samples of sample_kmers k-mers together
    bool one = false;
    SYL_TRY(scan_one_batch(ctx, n_samples, sample_kmers, n_samples ? (sample_kmers + n_samples - 1) / n_samples : 0, &one));
    *scan = plan_scan(ScanShape{n_kmers, n_tracked, n_genomes, n_samples, sample_kmers, one, false}) ? 1 : 0;
    return SYL_OK;
}

void syl_db_shards_free(syl_db_shards *s) {
    if (!s) return;
    if (s->pinned) cudaFreeHost(s->pinned);
    delete s;
}

}  // extern "C"
