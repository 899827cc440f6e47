// db_index.cu — the containment index of a database (syl_db): built from device or host sketches by bucket scatter,
// in bounded device memory (contain.hpp: bucket_of, DbInput).
#include <cub/cub.cuh>

#include <algorithm>
#include <new>
#include <vector>

#include "contain.hpp"
#include "ingest.hpp"

namespace syl {

// ---- index build ----------------------------------------------------------------------------
//
// The index is every entry (key, gid = genome << 1 | tracked) of the db in (key, tracked, genome) order: the order of a
// stable sort of all genomes' k-mers in genome order followed by all tracked k-mers in genome order (entries equal in
// key and gid cannot be told apart).  It is built without a global sort: a max pass fixes the bucket directory
// (bucket_of in contain.hpp), a histogram pass counts each bucket, a scatter pass writes every entry into its bucket's segment
// of the final arrays, and each bucket is then sorted on its own.  Every pass reads the input as CSR chunks
// (DbChunk): a device source is one chunk, a host source is cut into chunks that are copied while the previous
// chunk's kernels run, so the build needs device memory for the index and two staging chunks, not for a sort.

__global__ void k_glen(const uint64_t *__restrict__ kmer_off, uint64_t n_genomes, uint32_t *__restrict__ glen) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < n_genomes) glen[g] = (uint32_t)(kmer_off[g + 1] - kmer_off[g]);
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

static uint64_t db_chunk_entries() {  // SYL_DB_CHUNK overrides (tests; read per call)
    if (const char *e = getenv("SYL_DB_CHUNK")) {
        const long long v = atoll(e);
        if (v >= 1) return (uint64_t)v;
    }
    return 1ull << 25;
}

// Hands the input to a pass chunk by chunk.  A device source is one chunk over the whole arrays.  A host source is
// cut into chunks of at most C entries and, per segment, at most min(C, G) genome offsets; each chunk is copied on the
// ctx's copy stream (ingest.hpp), straight from the caller's arrays, into one of two staging buffers while the previous
// chunk's kernels run on the ctx stream.
struct DbFeed {
    syl_ctx *ctx;
    const DbInput &in;
    uint64_t C = 0, L = 0;
    BuildBuf stage[2];
    SlotHandoff<2> handoff;  // after the staging buffers (ingest.hpp); those are not cached blocks, so no fence
    DbFeed(syl_ctx *c, const DbInput &i) : ctx(c), in(i), stage{BuildBuf(c), BuildBuf(c)} {}
    int init() {
        if (in.mem == SYL_MEM_DEVICE) return SYL_OK;
        C = std::min<uint64_t>(db_chunk_entries(), in.n[0] + in.n[1]);
        L = std::min<uint64_t>(C, in.G);
        cudaStream_t cs = nullptr;
        SYL_TRY(ctx_copy_stream(ctx, &cs));
        SYL_TRY(handoff.init(cs, ctx->stream));
        for (int b = 0; b < 2; b++) SYL_TRY(stage[b].alloc((C + 2 * L) * 8));
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
            SYL_TRY(handoff.before_copy(b));
            uint64_t *kw = stage[b].as<uint64_t>(), *ow = kw + C;
            DbChunk c{};
            for (int s = 0; s < ns; s++) {
                const uint64_t n = p1[s] - p0[s], no = ghi[s] - glo[s] + 1;
                SYL_CUDA(cudaMemcpyAsync(kw, in.keys[part[s]] + p0[s], n * 8, cudaMemcpyHostToDevice, handoff.cs));
                SYL_CUDA(cudaMemcpyAsync(ow, in.off[part[s]] + glo[s], no * 8, cudaMemcpyHostToDevice, handoff.cs));
                c.keys[s] = kw; c.off[s] = ow; c.n_off[s] = no; c.g0[s] = glo[s]; c.p0[s] = p0[s]; c.n[s] = n; c.part[s] = part[s];
                kw += n;
                ow += no;
            }
            SYL_TRY(handoff.copied_in(b));
            SYL_TRY(handoff.take(b));
            launch(c);
            ctx->launches++;
            SYL_CUDA(cudaGetLastError());
            SYL_TRY(handoff.done(b));
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

// CSR offsets of G genomes (or samples) in host memory (tracked_off may be NULL): the chunk planner and the scatter's
// genome search walk them, so they must start at 0 and never decrease
int check_host_offsets(const uint64_t *kmer_off, const uint64_t *tracked_off, uint64_t G) {
    for (const uint64_t *o : {kmer_off, tracked_off}) {
        if (!o) continue;
        bool bad = o[0] != 0;
        for (uint64_t i = 1; i <= G && !bad; i++) bad = o[i] < o[i - 1];
        if (bad) { set_error(BAD_OFFSETS); return SYL_ERR_ARG; }
    }
    return SYL_OK;
}

int check_db_size(uint64_t nk, uint64_t nt, uint64_t G) {
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
int db_build(syl_ctx *ctx, const DbInput &in, const uint64_t *gn_size, int has_tracked, int k, uint64_t c,
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

}  // extern "C"
