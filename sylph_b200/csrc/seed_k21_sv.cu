// k_seed<K=21, EMIT=0> for run lengths 24 / 30 / 32, ASCII and 2-bit input (EMIT 0: 16-byte survivors, 1: 32-byte read-sketch events)
#include "seed_kernel.cuh"

namespace syl {
SEED_DEFINE_KERNELS(seed_kernels_k21_sv, 21, 0)
}  // namespace syl
