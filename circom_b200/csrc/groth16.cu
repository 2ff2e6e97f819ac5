// Groth16 proof assembly kernel and its launcher (see groth16.h).  Product code: part of libcircom_b200.so.
#define CW_KERNELS_TAPE_ONLY 1
#define CW_MSM_NO_G1_KERNELS 1
#define CW_MSM_NO_G2_KERNELS 1
#define CW_GROTH16_KERNELS 1
#include "groth16.cuh"
#include "groth16.h"

namespace cw {

static_assert(sizeof(Groth16Consts) == 4 * G16_CONSTS_WORDS, "Groth16Consts layout");

cudaError_t groth16_set_params(const FrParams *table, size_t bytes) { return cudaMemcpyToSymbol(c_fr, table, bytes); }

void groth16_launch_assemble(const void *consts, const uint64_t *ma, const uint64_t *mb1, const uint64_t *mb2,
                             const uint64_t *mc, const uint64_t *mh, const uint64_t *rs, uint32_t count, uint64_t *proofs,
                             cudaStream_t stream) {
    const dim3 grid((count + G16_THREADS - 1) / G16_THREADS, 2);
    groth16_assemble_kernel<<<grid, G16_THREADS, 0, stream>>>((const Groth16Consts *)consts, (const u32 *)ma, (const u32 *)mb1,
                                                             (const u32 *)mb2, (const u32 *)mc, (const u32 *)mh, (const u32 *)rs,
                                                             count, (u32 *)proofs);
}

}  // namespace cw
