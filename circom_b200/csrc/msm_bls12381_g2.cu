// BLS12-381 G2 multi-scalar multiplication kernels and their launchers (see msm_bls12381_g2.h).  Product code: part of
// libcircom_b200.so.
#define CW_KERNELS_TAPE_ONLY 1
#define CW_MSM_NO_G1_KERNELS 1
#define CW_MSM_NO_BLS_G1_KERNELS 1
#include "msm_bls12381_g2.cuh"
#include "msm_bls12381_g2.h"

namespace cw {

static_assert(sizeof(XyzzG2_381) == MSM_BLS_G2_POINT_BYTES, "BLS12-381 G2 bucket size");

cudaError_t msm_bls12381_g2_set_params() {
    const Fp381Params h = fp381_params();
    return cudaMemcpyToSymbol(c_fp381_g2, &h, sizeof(h));
}

int bls12381_g2_point_mont(const uint64_t *xy, u32 *mont, int *bad_coef) {
    static const Fp381Params P = fp381_params();
    u32 canon[48];
    memcpy(canon, xy, 192);
    return bls12381_g2_to_mont(mont, canon, bad_coef, P);
}

void msm_bls12381_g2_launch_runs(bool affine, const u32 *keys, const u32 *vals, const u32 *bases, const void *pts,
                                 uint64_t N, u32 c, void *buckets, u32 *okeys, void *opts, cudaStream_t stream) {
    const uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN;
    const u32 grid = (u32)((threads + MSM_BLS_G2_THREADS - 1) / MSM_BLS_G2_THREADS);
    if (affine)
        msm_bls_g2_runs_kernel<true><<<grid, MSM_BLS_G2_THREADS, 0, stream>>>(keys, vals, bases, nullptr, N, c,
                                                                              (XyzzG2_381 *)buckets, okeys, (XyzzG2_381 *)opts);
    else
        msm_bls_g2_runs_kernel<false><<<grid, MSM_BLS_G2_THREADS, 0, stream>>>(keys, nullptr, nullptr, (const XyzzG2_381 *)pts,
                                                                               N, c, (XyzzG2_381 *)buckets, okeys,
                                                                               (XyzzG2_381 *)opts);
}

void msm_bls12381_g2_launch_reduce(const void *buckets, u32 B, u32 n_win, void *segs, void *wins, u32 W, u32 c, u32 count,
                                   uint4 *out, cudaStream_t stream) {
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    const uint64_t seg_threads = (uint64_t)n_win * per;
    msm_bls_g2_segments_kernel<<<(u32)((seg_threads + MSM_BLS_G2_THREADS - 1) / MSM_BLS_G2_THREADS), MSM_BLS_G2_THREADS, 0,
                                 stream>>>((const XyzzG2_381 *)buckets, B, n_win, (XyzzG2_381 *)segs);
    msm_bls_g2_windows_kernel<<<n_win, MSM_BLS_G2_WIN_THREADS, 0, stream>>>((const XyzzG2_381 *)segs, per, (XyzzG2_381 *)wins);
    msm_bls_g2_final_kernel<<<(count + MSM_BLS_G2_THREADS - 1) / MSM_BLS_G2_THREADS, MSM_BLS_G2_THREADS, 0, stream>>>(
        (const XyzzG2_381 *)wins, W, c, count, out);
}

}  // namespace cw
