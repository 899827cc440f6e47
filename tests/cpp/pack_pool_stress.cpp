// Scheduler stress test of syl::PackPool without a GPU: mirrors the packed chunk loop of feed_host (sample.cu) —
// packed chunks in order from the front behind a gate of R staging slots, chunks taken over by the caller from the
// back, forced alternation (SYL_INGEST_FORCE_STEAL).  Must terminate.
#include "host_pack.hpp"
#include <cstdio>
#include <cstdlib>
#include <chrono>
using namespace syl;
int main() {
    PackPool pool(6);
    for (int rep = 0; rep < 200; rep++) {
        const int R = 4;
        const size_t nch = 1 + rand() % 40;
        std::vector<std::vector<uint8_t>> src(nch);
        std::vector<std::vector<uint32_t>> dst(R);
        std::vector<PackItem> items; std::vector<uint32_t> ci(nch);
        for (int s = 0; s < R; s++) dst[s].resize(1 << 14);
        for (size_t c = 0; c < nch; c++) {
            src[c].assign(16 * (1 + rand() % 4000), 'C');
            uint32_t n = 0;
            for (size_t o = 0; o < src[c].size(); o += 4096, n++) items.push_back({src[c].data() + o, std::min<size_t>(4096, src[c].size() - o), dst[c % R].data() + o / 16, nullptr, 0, 0, nullptr, (uint32_t)c});
            ci[c] = n;
        }
        pool.start(&items, &ci, R - 1);
        int64_t f = 0, bk = (int64_t)nch - 1, last = -1; size_t na = 0, np = 0; bool force = rep % 2; bool turn = true;
        while (f <= bk) {
            bool sf = force && turn;
            if (!sf && pool.chunk_done((uint32_t)f)) { if (last >= 0) pool.open_gate(last + R); last = f; f++; np++; turn = true; continue; }
            if (bk > f && ((force && turn) || (!force && rand() % 3 == 0)) && pool.try_skip_chunk((uint32_t)bk)) { na++; bk--; turn = false; continue; }
            if (sf) { turn = false; continue; }
            pool.wait_chunk((uint32_t)f);
        }
        pool.open_gate((int64_t)1 << 60);
        pool.finish();
    }
    printf("ok\n");
    return 0;
}
