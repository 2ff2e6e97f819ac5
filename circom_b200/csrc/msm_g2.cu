// G2 multi-scalar multiplication kernels and their launchers (see msm_g2.h).  Product code: part of libcircom_b200.so.
#define CW_KERNELS_TAPE_ONLY 1
#define CW_MSM_NO_G1_KERNELS 1
#include "msm_g2.cuh"
#include "msm_g2.h"

namespace cw {

static_assert(sizeof(XyzzG2) == MSM_G2_POINT_BYTES, "G2 bucket size");

cudaError_t msm_g2_set_params(const FrParams *table, size_t bytes) { return cudaMemcpyToSymbol(c_fr, table, bytes); }

void msm_g2_launch_runs(bool affine, const u32 *keys, const u32 *vals, const u32 *bases, const void *pts, uint64_t N, u32 c,
                        void *buckets, u32 *okeys, void *opts, cudaStream_t stream) {
    const uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN;
    const u32 grid = (u32)((threads + MSM_G2_THREADS - 1) / MSM_G2_THREADS);
    if (affine)
        msm_g2_runs_kernel<true><<<grid, MSM_G2_THREADS, 0, stream>>>(keys, vals, bases, nullptr, N, c, (XyzzG2 *)buckets, okeys,
                                                                     (XyzzG2 *)opts);
    else
        msm_g2_runs_kernel<false><<<grid, MSM_G2_THREADS, 0, stream>>>(keys, nullptr, nullptr, (const XyzzG2 *)pts, N, c,
                                                                      (XyzzG2 *)buckets, okeys, (XyzzG2 *)opts);
}

void msm_g2_launch_reduce(const void *buckets, u32 B, u32 n_win, void *segs, void *wins, u32 W, u32 c, u32 count, uint4 *out,
                          cudaStream_t stream) {
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    const uint64_t seg_threads = (uint64_t)n_win * per;
    msm_g2_segments_kernel<<<(u32)((seg_threads + MSM_G2_THREADS - 1) / MSM_G2_THREADS), MSM_G2_THREADS, 0, stream>>>(
        (const XyzzG2 *)buckets, B, n_win, (XyzzG2 *)segs);
    msm_g2_windows_kernel<<<n_win, MSM_G2_THREADS, 0, stream>>>((const XyzzG2 *)segs, per, (XyzzG2 *)wins);
    msm_g2_final_kernel<<<(count + MSM_G2_THREADS - 1) / MSM_G2_THREADS, MSM_G2_THREADS, 0, stream>>>((const XyzzG2 *)wins, W, c,
                                                                                                     count, out);
}

}  // namespace cw
