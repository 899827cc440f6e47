// Scratch microbenchmark: the seeding hot loop alone (no staging, packing, tables or output) at several
// occupancies, to separate "what the instruction mix can sustain" from "what the phases around it cost".
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --expt-relaxed-constexpr -o exp/hotloop_bench scripts/hotloop_bench.cu
#include <cstdio>
#include <vector>
#include "../sylph_b200/csrc/seed_kernel.cuh"

using namespace syl;
namespace syl { void set_error(const std::string &) {} thread_local syl_ctx *tl_ctx = nullptr; }

// diagnostic variants of the loop body: which part of the per-window work costs what
//   MODE 0 full (seed_run, the loop k_seed runs)   1 hash only (operands from registers)   2 extraction + hash of the forward k-mer (no canonical)
//   3 full, canonical by 64-bit integer compare   4 full, FP64 compare + SEL instead of predicated IMAD
template <int K, int W, int MODE>
__device__ __forceinline__ uint32_t run_variant(const uint32_t *fw, const uint32_t *cwp, int p, uint32_t thr_hi, const ImadConst ic) {
    if (MODE == 0) return seed_run<K, W>(fw, cwp, p, thr_hi, ic);
    constexpr uint32_t PAD = 64 - 2 * K;
    constexpr uint32_t HI_MASK = (1u << (32 - PAD)) - 1u;
    uint32_t F[4], G[4];
    {
        const uint32_t bitpos = 32u + 2u * (uint32_t)p - PAD;
        const uint32_t q0 = bitpos >> 5, sh = bitpos & 31u;
        const uint32_t w0 = fw[q0], w1 = fw[q0 + 1], w2 = fw[q0 + 2], w3 = fw[q0 + 3], w4 = fw[q0 + 4];
        F[0] = __funnelshift_l(w1, w0, sh); F[1] = __funnelshift_l(w2, w1, sh); F[2] = __funnelshift_l(w3, w2, sh); F[3] = __funnelshift_l(w4, w3, sh);
        const uint32_t cq = (uint32_t)p >> 4, csh = ((uint32_t)p & 15u) * 2u;
        const uint32_t c0 = cwp[cq], c1 = cwp[cq + 1], c2 = cwp[cq + 2], c3 = cwp[cq + 3], c4 = cwp[cq + 4];
        G[0] = __funnelshift_r(c0, c1, csh); G[1] = __funnelshift_r(c1, c2, csh); G[2] = __funnelshift_r(c2, c3, csh); G[3] = __funnelshift_r(c3, c4, csh);
    }
    uint32_t cand = 0u;
#pragma unroll
    for (int i = 0; i < W; i++) {
        const int jb = (2 * i) >> 5;
        const uint32_t sft = (uint32_t)((2 * i) & 31);
        uint32_t c_lo, c_hi;
        if (MODE == 1) {
            c_lo = F[i & 3] + (uint32_t)i * 0x9E3779B9u; c_hi = G[i & 3];
        } else {
            const uint32_t f_hi = __funnelshift_l(F[jb + 1], F[jb], sft) & HI_MASK;
            const uint32_t f_lo = __funnelshift_l(F[jb + 2], F[jb + 1], sft);
            if (MODE == 2) { c_lo = f_lo; c_hi = f_hi; }
            else {
                const uint32_t r_lo = __funnelshift_r(G[jb], G[jb + 1], sft);
                const uint32_t r_hi = __funnelshift_r(G[jb + 1], G[jb + 2], sft) & HI_MASK;
                if (MODE == 3) {
                    const uint64_t f = ((uint64_t)f_hi << 32) | f_lo, rr = ((uint64_t)r_hi << 32) | r_lo;
                    const uint64_t canon = f < rr ? f : rr;
                    c_lo = (uint32_t)canon; c_hi = (uint32_t)(canon >> 32);
                } else {
                    asm("{\n\t.reg .pred p;\n\t.reg .f64 a, b;\n\tmov.b64 a, {%2, %3};\n\tmov.b64 b, {%4, %5};\n\t"
                        "setp.lt.f64 p, a, b;\n\tselp.b32 %0, %2, %4, p;\n\tselp.b32 %1, %3, %5, p;\n\t}"
                        : "=r"(c_lo), "=r"(c_hi) : "r"(f_lo), "r"(f_hi), "r"(r_lo), "r"(r_hi));
                }
            }
        }
        const uint32_t hh = hash_hi32(c_lo, c_hi);
        asm("{\n\t.reg .pred p;\n\tsetp.le.u32 p, %1, %2;\n\t@p mad.lo.u32 %0, %3, %4, %0;\n\t}"
            : "+r"(cand) : "r"(hh), "r"(thr_hi), "r"(ic.one), "r"(1u << i));
    }
    return cand;
}

template <int W, int MODE>
__global__ void __launch_bounds__(256) k_hot(uint32_t *out, int iters, ImadConst ic, uint32_t thr_hi) {
    extern __shared__ uint32_t sm[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t *fw = sm + wid * 640, *cw = fw + 320;   // 320 words = 5120 bases per stream per warp
    for (int i = lane; i < 640; i += 32) fw[i] = (uint32_t)(i * 2654435761u) ^ (blockIdx.x * 40503u) ^ (uint32_t)(wid << 20);
    __syncwarp();
    uint32_t acc = 0;
    int p = lane * W;
    for (int it = 0; it < iters; it++) {
        acc ^= run_variant<31, W, MODE>(fw, cw, p, thr_hi, ic);
        p += 32 * W;
        if (p > 4096) p -= 4096;
    }
    out[blockIdx.x * 256 + threadIdx.x] = acc;
}

int main() {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    const int sms = prop.multiProcessorCount;
    uint32_t *out; cudaMalloc(&out, (size_t)sms * 8 * 256 * 4 * 2);
    const ImadConst ic = {{0u, 0u, 0u}, 1u, 0u};
    const uint32_t thr_hi = 0x0147AE14u;
    const int iters = 2000;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("device %s, %d SMs\n", prop.name, sms);
    typedef void (*kern_t)(uint32_t *, int, ImadConst, uint32_t);
    struct V { const char *name; kern_t k; int W; };
    const V vs[] = {{"W=30 full", k_hot<30, 0>, 30}, {"W=32 full", k_hot<32, 0>, 32}, {"W=30 hash only", k_hot<30, 1>, 30},
                    {"W=30 extract fwd + hash (no canonical)", k_hot<30, 2>, 30}, {"W=30 full, integer compare", k_hot<30, 3>, 30},
                    {"W=30 full, FP64 compare + SEL", k_hot<30, 4>, 30}};
    for (const V &v : vs) {
        cudaFuncSetAttribute(v.k, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        for (int ctas : {2, 3, 4}) {
            size_t smem = (size_t)(220 * 1024) / ctas;
            smem = smem / 128 * 128;
            const int grid = sms * ctas;
            float best = 1e9f;
            for (int rep = 0; rep < 4; rep++) {
                cudaEventRecord(e0);
                v.k<<<grid, 256, smem>>>(out, iters, ic, thr_hi);
                cudaEventRecord(e1);
                cudaEventSynchronize(e1);
                float ms; cudaEventElapsedTime(&ms, e0, e1);
                if (ms < best) best = ms;
            }
            const double windows = (double)grid * 256 * iters * v.W;
            const double rate = windows / (best * 1e-3);
            printf("%-44s %2d warps/SM: %.3f T windows/s = %.1f cycles per warp-window at 1.965 GHz; 0.8e9 windows in %.3f ms\n", v.name, ctas * 8,
                   rate / 1e12, 1.965e9 * sms * 4 * 32 / rate, 0.8e9 / rate * 1e3);
        }
    }
    cudaError_t e = cudaDeviceSynchronize();
    printf("status: %s\n", cudaGetErrorString(e));
    return 0;
}
