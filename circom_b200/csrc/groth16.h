// The Groth16 assembly kernel (groth16.cuh) lives in its own translation unit, groth16.cu, like the G2 MSM kernels:
// capi.cu reads the proving key, runs the quotient and the five MSMs and calls this launcher for the last step.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "fr_device.cuh"

namespace cw {
// u32 words of Groth16Consts (groth16.cuh): alpha1, beta1, delta1 (16 each), beta2, delta2 (32 each), Montgomery images
constexpr size_t G16_CONSTS_WORDS = 112;
// this unit's copy of the constant field-parameter table
cudaError_t groth16_set_params(const FrParams *table, size_t bytes);
// proofs [count][32] u64 canonical from the MSM results and (r, s) (layouts: groth16_assemble_kernel); consts: a device
// Groth16Consts
void groth16_launch_assemble(const void *consts, const uint64_t *ma, const uint64_t *mb1, const uint64_t *mb2,
                             const uint64_t *mc, const uint64_t *mh, const uint64_t *rs, uint32_t count, uint64_t *proofs,
                             cudaStream_t stream);
}  // namespace cw
