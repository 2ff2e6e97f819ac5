// The BLS12-381 G2 multi-scalar multiplication kernels (msm_bls12381_g2.cuh) live in their own translation unit,
// msm_bls12381_g2.cu, with their own constant parameter record.  capi.cu checks the bases with bls12381_g2_point_mont,
// plans the scratch, runs the digits and the sort (msm.cuh), and calls these launchers for the rest.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "fr_device.cuh"

namespace cw {
constexpr size_t MSM_BLS_G2_POINT_BYTES = 384;   // sizeof(XyzzG2_381)
// this unit's constant Fp381Params
cudaError_t msm_bls12381_g2_set_params();
// one canonical affine point (x.c0, x.c1, y.c0, y.c1: 6 u64 each) to the Montgomery [48] u32 the kernels read: 0, or 1
// when a coefficient is not below q (*bad_coef: its index 0..3), 2 when the point is not on y^2 = x^3 + 4 (1 + u).  All
// zeros is infinity and stays zero.  Host code.
int bls12381_g2_point_mont(const uint64_t *xy, u32 *mont, int *bad_coef);
// one run-summing level: over the sorted affine items (affine: keys, vals, bases [n][48] u32) or over the partial sums of
// the level before (keys, pts)
void msm_bls12381_g2_launch_runs(bool affine, const u32 *keys, const u32 *vals, const u32 *bases, const void *pts,
                                 uint64_t N, u32 c, void *buckets, u32 *okeys, void *opts, cudaStream_t stream);
// buckets [n_win][B] -> segment sums -> window sums -> Horner's rule and affine canonical out [count][2][2][6] u64
void msm_bls12381_g2_launch_reduce(const void *buckets, u32 B, u32 n_win, void *segs, void *wins, u32 W, u32 c, u32 count,
                                   uint4 *out, cudaStream_t stream);
}  // namespace cw
