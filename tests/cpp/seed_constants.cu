// seed_constants.cu — prints the seeding kernel's geometry (seed_kernel.cuh) for tests/seed_scripts.py, so that the
// scripted seeding batches place their edges where the kernel compiled with the same definitions has them.
// Host-only: nothing here runs on a GPU.
#include "seed_kernel.cuh"

int main() {
    printf("SEED_TILE %d\nSEED_THREADS %d\nSEED_HALO %d\nSEED_STAGE %d\nSEED_CAND %d\nSEED_W_MIN %d\nSEED_W_MAX %d\n"
           "SEED_MAXRUNS %d\nSEED_NCHUNK16 %d\nSEED_PK_WORDS %d\n",
           syl::SEED_TILE, syl::SEED_THREADS, syl::SEED_HALO, syl::SEED_STAGE, syl::SEED_CAND, syl::SEED_W_MIN,
           syl::SEED_W_MAX, syl::SEED_MAXRUNS, syl::SEED_NCHUNK16, syl::SEED_PK_WORDS);
    return 0;
}
