// The G2 multi-scalar multiplication kernels (msm_g2.cuh) live in their own translation unit, msm_g2.cu: their point type
// is four times G1's, and keeping them out of capi.cu keeps that unit's ptxas time as it was.  capi.cu plans the scratch,
// runs the digits and the sort (msm.cuh), and calls these launchers for the rest.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "fr_device.cuh"

namespace cw {
constexpr size_t MSM_G2_POINT_BYTES = 256;   // sizeof(XyzzG2)
// this unit's copy of the constant field-parameter table (every .cu has its own c_fr without relocatable device code)
cudaError_t msm_g2_set_params(const FrParams *table, size_t bytes);
// one run-summing level: over the sorted affine items (affine: keys, vals, bases [n][32] u32) or over the partial sums of
// the level before (keys, pts)
void msm_g2_launch_runs(bool affine, const u32 *keys, const u32 *vals, const u32 *bases, const void *pts, uint64_t N, u32 c,
                        void *buckets, u32 *okeys, void *opts, cudaStream_t stream);
// buckets [n_win][B] -> segment sums -> window sums -> Horner's rule and affine canonical out [count][2][2][4] u64
void msm_g2_launch_reduce(const void *buckets, u32 B, u32 n_win, void *segs, void *wins, u32 W, u32 c, u32 count, uint4 *out,
                          cudaStream_t stream);
}  // namespace cw
