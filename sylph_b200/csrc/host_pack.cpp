// host_pack.cpp — exact BYTE_TO_SEQ (src/types.rs:50-59) 2-bit packing on the host + the worker pool
// that feeds the pinned staging ring of syl_sketch_reads (host-memory inputs).  Compiled by g++ (no
// CUDA in here); AVX2 path selected at run time, scalar table path otherwise.
#include "host_pack.hpp"

#include <immintrin.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>

#include <algorithm>

namespace syl {

namespace {

constexpr uint64_t PACK_PREFETCH_DEFAULT = 2048;  // bytes the packer prefetches ahead of its read position

struct Lut {
    uint8_t t[256];
    Lut() {
        memset(t, 0, sizeof(t));
        t[1] = 1; t[2] = 2; t[3] = 3;
        t['C'] = t['c'] = 1;
        t['G'] = t['g'] = 2;
        t['T'] = t['t'] = t['U'] = t['u'] = 3;
    }
};
const Lut g_lut;

inline uint32_t pack16_scalar(const uint8_t *p) {
    uint32_t w = 0;
    for (int j = 0; j < 16; j++) w = (w << 2) | g_lut.t[p[j]];
    return w;
}

void pack2_scalar(const uint8_t *bases, uint64_t n, uint32_t *words) {
    const uint64_t full = n / 16;
    for (uint64_t w = 0; w < full; w++) words[w] = pack16_scalar(bases + 16 * w);
    if (n % 16) {
        uint8_t tmp[16] = {0};
        memcpy(tmp, bases + 16 * full, n % 16);
        words[full] = pack16_scalar(tmp);
    }
}

// 32 bases -> 2 words.  Byte class by two nibble tables ANDed together: bit a = {C,c}, b = {0x01},
// c = {G,g}, d = {0x02}, e = {T,t,U,u}, f = {0x03}; code bit 0 = a|b|e|f, code bit 1 = c|d|e|f.
__attribute__((target("avx2"))) void pack2_avx2(const uint8_t *bases, uint64_t n, uint32_t *words) {
    const __m256i lo_tab = _mm256_setr_epi8(0, 0x02, 0x08, 0x21, 0x10, 0x10, 0, 0x04, 0, 0, 0, 0, 0, 0, 0, 0,
                                            0, 0x02, 0x08, 0x21, 0x10, 0x10, 0, 0x04, 0, 0, 0, 0, 0, 0, 0, 0);
    // hi nibble 0: b,d,f ; 4,6: a,c ; 5,7: e
    const __m256i hi_tab = _mm256_setr_epi8(0x2A, 0, 0, 0, 0x05, 0x10, 0x05, 0x10, 0, 0, 0, 0, 0, 0, 0, 0,
                                            0x2A, 0, 0, 0, 0x05, 0x10, 0x05, 0x10, 0, 0, 0, 0, 0, 0, 0, 0);
    const __m256i nib = _mm256_set1_epi8(0x0F);
    const __m256i m_b0 = _mm256_set1_epi8(0x33);  // a|b|e|f  (0x01|0x02|0x10|0x20)
    const __m256i m_b1 = _mm256_set1_epi8(0x3C);  // c|d|e|f  (0x04|0x08|0x10|0x20)
    const __m256i zero = _mm256_setzero_si256();
    const __m256i one = _mm256_set1_epi8(1), two = _mm256_set1_epi8(2);
    const __m256i w41 = _mm256_set1_epi16(0x0104);      // bytes (4, 1): c0*4 + c1
    const __m256i w161 = _mm256_set1_epi32(0x00010010);  // words (16, 1): p0*16 + p1
    const __m256i gather = _mm256_setr_epi8(12, 8, 4, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1,
                                            12, 8, 4, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1);
    const uint64_t full = n / 32;
    for (uint64_t i = 0; i < full; i++) {
        const __m256i v = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(bases + 32 * i));
        const __m256i lo = _mm256_and_si256(v, nib);
        const __m256i hi = _mm256_and_si256(_mm256_srli_epi16(v, 4), nib);
        const __m256i m = _mm256_and_si256(_mm256_shuffle_epi8(lo_tab, lo), _mm256_shuffle_epi8(hi_tab, hi));
        const __m256i b0 = _mm256_andnot_si256(_mm256_cmpeq_epi8(_mm256_and_si256(m, m_b0), zero), one);
        const __m256i b1 = _mm256_andnot_si256(_mm256_cmpeq_epi8(_mm256_and_si256(m, m_b1), zero), two);
        const __m256i code = _mm256_or_si256(b0, b1);                   // one 2-bit code per byte
        const __m256i p2 = _mm256_maddubs_epi16(code, w41);            // 16-bit lanes: c0*4 + c1
        const __m256i p4 = _mm256_madd_epi16(p2, w161);                // 32-bit lanes: 4 bases, MSB-first, in the low byte
        const __m256i g = _mm256_shuffle_epi8(p4, gather);            // low dword of each 128-bit half = one word
        words[2 * i] = (uint32_t)_mm256_extract_epi32(g, 0);
        words[2 * i + 1] = (uint32_t)_mm256_extract_epi32(g, 4);
    }
    if (n % 32) pack2_scalar(bases + 32 * full, n % 32, words + 2 * full);
}

__attribute__((target("avx512f,avx512bw,avx512vbmi"), always_inline)) inline __m128i pack64_avx512(
    const uint8_t *src, __m512i tab_lo, __m512i tab_hi, __m512i w41, __m512i w161, __m128i rev) {
    const __m512i v = _mm512_loadu_si512(src);
    const __mmask64 hi = _mm512_movepi8_mask(v);                                // bytes >= 0x80 -> code 0
    const __m512i code = _mm512_maskz_permutex2var_epi8(~hi, tab_lo, v, tab_hi);  // BYTE_TO_SEQ[b & 0x7F]
    const __m512i p2 = _mm512_maddubs_epi16(code, w41);
    const __m512i p4 = _mm512_madd_epi16(p2, w161);                             // 16 dwords: 4 bases each, in the low byte
    return _mm_shuffle_epi8(_mm512_cvtepi32_epi8(p4), rev);                     // word = B0<<24 | B1<<16 | B2<<8 | B3
}

// 64 bases -> 4 words with AVX-512 VBMI: the low 7 bits of a byte index a 128-entry BYTE_TO_SEQ table held in two
// registers (VPERMI2B); bytes >= 0x80 are masked to 0.
__attribute__((target("avx512f,avx512bw,avx512vbmi"))) void pack2_avx512(const uint8_t *bases, uint64_t n, uint32_t *words) {
    alignas(64) uint8_t tlo[64], thi[64];
    for (int i = 0; i < 64; i++) { tlo[i] = g_lut.t[i]; thi[i] = g_lut.t[64 + i]; }
    const __m512i tab_lo = _mm512_load_si512(tlo), tab_hi = _mm512_load_si512(thi);
    const __m512i w41 = _mm512_set1_epi16(0x0104);       // bytes (4, 1): c0*4 + c1
    const __m512i w161 = _mm512_set1_epi32(0x00010010);  // words (16, 1): p0*16 + p1
    const __m128i rev = _mm_setr_epi8(3, 2, 1, 0, 7, 6, 5, 4, 11, 10, 9, 8, 15, 14, 13, 12);
    const uint64_t full = n / 64;
    // software prefetch distance in bytes (0 = off): the hardware streamer stops at every 4 KB page of the (pinned,
    // small-page) source buffer; SYL_PACK_PREFETCH overrides
    static const uint64_t pf = []() -> uint64_t { const char *e = getenv("SYL_PACK_PREFETCH"); return e ? (uint64_t)atoll(e) : PACK_PREFETCH_DEFAULT; }();
#define pack64(src) pack64_avx512((src), tab_lo, tab_hi, w41, w161, rev)
    uint64_t i = 0;
    for (; i + 4 <= full; i += 4) {  // 256 bases -> one 64-byte store
        const uint8_t *src = bases + 64 * i;
        if (pf) {
            _mm_prefetch(reinterpret_cast<const char *>(src + pf), _MM_HINT_T0);
            _mm_prefetch(reinterpret_cast<const char *>(src + pf + 64), _MM_HINT_T0);
            _mm_prefetch(reinterpret_cast<const char *>(src + pf + 128), _MM_HINT_T0);
            _mm_prefetch(reinterpret_cast<const char *>(src + pf + 192), _MM_HINT_T0);
        }
        __m512i o = _mm512_castsi128_si512(pack64(src));
        o = _mm512_inserti32x4(o, pack64(src + 64), 1);
        o = _mm512_inserti32x4(o, pack64(src + 128), 2);
        o = _mm512_inserti32x4(o, pack64(src + 192), 3);
        _mm512_storeu_si512(words + 4 * i, o);
    }
    for (; i < full; i++) _mm_storeu_si128(reinterpret_cast<__m128i *>(words + 4 * i), pack64(bases + 64 * i));
#undef pack64
    if (n % 64) pack2_scalar(bases + 64 * full, n % 64, words + 4 * full);
}

bool have_avx2() {
    static const bool v = __builtin_cpu_supports("avx2") && getenv("SYL_PACK_SCALAR") == nullptr;
    return v;
}
bool have_avx512() {
    static const bool v = __builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512bw") && __builtin_cpu_supports("avx512vbmi") &&
                          getenv("SYL_PACK_SCALAR") == nullptr && getenv("SYL_PACK_AVX2") == nullptr;
    return v;
}

}  // namespace

void pack2_range(const uint8_t *bases, uint64_t n_bases, uint32_t *words) {
    if (have_avx512()) pack2_avx512(bases, n_bases, words);
    else if (have_avx2()) pack2_avx2(bases, n_bases, words);
    else pack2_scalar(bases, n_bases, words);
}

int default_pack_threads() {
    if (const char *e = getenv("SYL_PACK_THREADS")) {
        const int v = atoi(e);
        if (v > 0) return std::min(v, 512);
    }
    unsigned hc = std::thread::hardware_concurrency();
    if (!hc) hc = 1;
    unsigned lw = 1;
    if (const char *e = getenv("LOCAL_WORLD_SIZE")) {  // one process per GPU (torchrun): share the host's cores
        const int v = atoi(e);
        if (v > 1) lw = (unsigned)v;
    }
    hc = std::max(1u, hc / lw);
    // a container's CPU quota (cgroup v2 cpu.max / v1 cfs_quota): threads beyond it only get the process throttled
    {
        long long quota = -1, period = 100000;
        if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
            char q[64] = {0};
            if (fscanf(f, "%63s %lld", q, &period) >= 1 && strcmp(q, "max") != 0) quota = atoll(q);
            fclose(f);
        } else if (FILE *g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
            if (fscanf(g, "%lld", &quota) != 1) quota = -1;
            fclose(g);
            if (FILE *h = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (fscanf(h, "%lld", &period) != 1) period = 100000; fclose(h); }
        }
        if (quota > 0 && period > 0) {  // the ranks share the quota; leave one core's worth for the threads that feed the GPUs
            const unsigned q = (unsigned)((quota + period - 1) / period);
            const unsigned mine = q > lw ? (q - 1) / lw : 1u;
            return (int)std::max(1u, std::min(std::min(hc, 32u), mine));
        }
    }
    // the packer is memory-bound well before all cores of a big host are busy
    return (int)std::max(1u, std::min(hc > 2 ? hc / 2u : hc, 32u));
}

PackPool::PackPool(int n_threads) {
    for (int i = 0; i < std::max(1, n_threads); i++) workers_.emplace_back([this]() { worker(); });
}

PackPool::~PackPool() {
    {
        std::lock_guard<std::mutex> lk(mu_);
        stop_ = true;
    }
    cv_work_.notify_all();
    for (auto &t : workers_) t.join();
}

void PackPool::start(const std::vector<PackItem> *items, const std::vector<uint32_t> *chunk_items, int64_t gate) {
    {
        std::lock_guard<std::mutex> lk(mu_);
        items_ = items;
        remaining_ = *chunk_items;
        taken_.assign(chunk_items->size(), 0);
        skipped_.assign(chunk_items->size(), 0);
        next_ = 0;
        done_ = 0;
        gate_ = gate;
    }
    cv_work_.notify_all();
}

void PackPool::open_gate(int64_t gate) {
    {
        std::lock_guard<std::mutex> lk(mu_);
        if (gate > gate_) gate_ = gate;
    }
    cv_work_.notify_all();
}

void PackPool::worker() {
    std::unique_lock<std::mutex> lk(mu_);
    for (;;) {
        cv_work_.wait(lk, [&]() {
            return stop_ || (items_ && next_ < items_->size() && (int64_t)(*items_)[next_].chunk <= gate_);
        });
        if (stop_) return;
        const PackItem it = (*items_)[next_++];
        taken_[it.chunk]++;
        if (!skipped_[it.chunk]) {
            lk.unlock();
            if (it.src) {
                pack2_range(it.src, it.n, it.dst);
            } else {
                for (uint64_t j = 0; j < it.off_n; j++) it.off_dst[j] = (uint32_t)(it.off_src[j] - it.off_base);
            }
            lk.lock();
        }
        done_++;
        if (--remaining_[it.chunk] == 0 || done_ == items_->size()) cv_done_.notify_all();
    }
}

void PackPool::wait_chunk(uint32_t c) {
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [&]() { return remaining_[c] == 0; });
}

bool PackPool::wait_chunk_for(uint32_t c, unsigned usec) {
    std::unique_lock<std::mutex> lk(mu_);
    return cv_done_.wait_for(lk, std::chrono::microseconds(usec), [&]() { return remaining_[c] == 0; });
}

bool PackPool::chunk_done(uint32_t c) {
    std::lock_guard<std::mutex> lk(mu_);
    return remaining_[c] == 0 && !skipped_[c];
}

bool PackPool::try_skip_chunk(uint32_t c) {
    std::lock_guard<std::mutex> lk(mu_);
    if (taken_[c] != 0 || skipped_[c]) return false;
    skipped_[c] = 1;
    return true;
}

void PackPool::finish() {
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [&]() { return !items_ || done_ == items_->size(); });
    items_ = nullptr;
}

}  // namespace syl
