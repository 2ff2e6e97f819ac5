// Groth16 proof assembly on BN254: the last step of a prover, after the five multi-scalar multiplications.  Per proof,
// with MA, MB1, MB2, MC, MH the MSM results and (r, s) the blinding scalars:
//   A  = alpha1 + MA + r delta1
//   B1 = beta1 + MB1 + s delta1           (only C reads it)
//   B2 = beta2 + MB2 + s delta2           (the proof's B)
//   C  = MC + MH + s A + r (beta1 + MB1)
// The last line equals snarkjs' MC + MH + s A + r B1 - r s delta1 (expand B1) and needs no r s product; its two
// variable-base products share one chain of doublings (Straus).  The point formulas are msm.cuh's / msm_g2.cuh's XYZZ
// ones, complete for the exceptional cases (equal points double, opposite points cancel, infinity).
//
// Host and device, like msm.cuh: tests/hostsim/groth16_sim.cpp runs these functions on the CPU.  The kernel (CUDA builds,
// groth16.cu) runs one thread per (proof, group): blockIdx.y = 0 computes A and C on G1, blockIdx.y = 1 computes B on G2.
#pragma once
#include "msm_g2.cuh"

namespace cw {

// the proving key's fixed points, Montgomery images mod q; all zeros = infinity
struct alignas(16) Groth16Consts {
    u32 alpha1[16], beta1[16], delta1[16];   // G1: x, y
    u32 beta2[32], delta2[32];               // G2: x.c0, x.c1, y.c0, y.c1
};

// The chains below are out-of-line functions, so that each group's addition and doubling formulas are compiled once
// per kernel rather than once per use.
#if defined(__CUDACC__)
#define G16_FN __host__ __device__ __noinline__
#else
#define G16_FN inline
#endif

// affine (x, y) -> XYZZ with ZZ = ZZZ = 1 (zeros: infinity); canonical coordinates are converted, Montgomery ones kept
G16_FN void g16_load(Xyzz &p, const u32 *xy, bool mont, const FrParams &P) {
    ntt_ld8(p.x, xy);
    ntt_ld8(p.y, xy + 8);
    if (u256_is_zero(p.x) && u256_is_zero(p.y)) {
        xyzz_inf(p);
        return;
    }
    if (!mont) {
        fr_to_mont(p.x, p.x, P);
        fr_to_mont(p.y, p.y, P);
    }
    u256_set(p.zz, P.r1);
    u256_set(p.zzz, P.r1);
}
G16_FN void g16_load(XyzzG2 &p, const u32 *xy, bool mont, const FrParams &P) {
    msm_ld_fq2(p.x, xy);
    msm_ld_fq2(p.y, xy + 16);
    if (fq2_is_zero(p.x) && fq2_is_zero(p.y)) {
        xyzz_inf(p);
        return;
    }
    if (!mont)
        for (u32 *c : {p.x.c0, p.x.c1, p.y.c0, p.y.c1}) fr_to_mont(c, c, P);
    u256_set(p.zz.c0, P.r1);
    u256_set_u32(p.zz.c1, 0);
    u256_set(p.zzz.c0, P.r1);
    u256_set_u32(p.zzz.c1, 0);
}

CW_HD u32 g16_bit(const u32 *k, int i) { return k ? (k[i >> 5] >> (i & 31)) & 1u : 0u; }

// acc = pts[0] + pts[1] + a p + b q for 256-bit a, b (NULL: zero).  One chain of doublings from the top bit adds p, q or
// p + q per bit (Straus); the sum of pts comes last, through the same addition.
template <class Pt>
G16_FN void g16_lincomb(Pt &acc, const Pt *pts, const Pt &p, const u32 *a, const Pt &q, const u32 *b, const FrParams &P) {
    Pt tab[4];                          // p, q, p + q, pts[0] + pts[1]
    tab[0] = p;
    tab[1] = q;
    tab[2] = p;
    tab[3] = pts[0];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int k = 2; k < 4; ++k) xyzz_add(tab[k], k == 2 ? q : pts[1], P);
    xyzz_inf(acc);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int i = 255; i >= -1; --i) {   // (i = -1: the sum of pts, without a doubling)
        if (i >= 0 && !xyzz_is_inf(acc)) xyzz_dbl(acc, P);
        const u32 sel = i >= 0 ? (g16_bit(a, i) | g16_bit(b, i) << 1) : 4u;
        if (sel) xyzz_add(acc, tab[sel - 1], P);
    }
}

G16_FN void g16_store(u32 *out, const Xyzz &p, const FrParams &P) {
    u32 x[8], y[8];
    xyzz_to_affine(x, y, p, P);
    fr_from_mont(out, x, P);
    fr_from_mont(out + 8, y, P);
}
G16_FN void g16_store(u32 *out, const XyzzG2 &p, const FrParams &P) {
    Fq2 x, y;
    xyzz_to_affine(x, y, p, P);
    fr_from_mont(out, x.c0, P);
    fr_from_mont(out + 8, x.c1, P);
    fr_from_mont(out + 16, y.c0, P);
    fr_from_mont(out + 24, y.c1, P);
}

// A and C of one proof (canonical affine [2][8] u32 each) from the canonical MSM results and the canonical r, s
G16_FN void groth16_g1(u32 *a_out, u32 *c_out, const Groth16Consts &K, const u32 *ma, const u32 *mb1, const u32 *mc,
                       const u32 *mh, const u32 *r, const u32 *s, const FrParams &P) {
    Xyzz pts[2], d, z, a, b1, c;
    xyzz_inf(z);
    g16_load(pts[0], K.alpha1, true, P);
    g16_load(pts[1], ma, false, P);
    g16_load(d, K.delta1, true, P);
    g16_lincomb(a, pts, d, r, z, nullptr, P);      // A = alpha1 + MA + r delta1
    g16_store(a_out, a, P);
    g16_load(pts[0], K.beta1, true, P);
    g16_load(pts[1], mb1, false, P);
    g16_lincomb(b1, pts, z, nullptr, z, nullptr, P);   // beta1 + MB1
    g16_load(pts[0], mc, false, P);
    g16_load(pts[1], mh, false, P);
    g16_lincomb(c, pts, a, s, b1, r, P);           // C = MC + MH + s A + r (beta1 + MB1)
    g16_store(c_out, c, P);
}

// B of one proof (canonical affine [2][2][8] u32: x.c0, x.c1, y.c0, y.c1)
G16_FN void groth16_g2(u32 *b_out, const Groth16Consts &K, const u32 *mb2, const u32 *s, const FrParams &P) {
    XyzzG2 pts[2], d, z, b;
    xyzz_inf(z);
    g16_load(pts[0], K.beta2, true, P);
    g16_load(pts[1], mb2, false, P);
    g16_load(d, K.delta2, true, P);
    g16_lincomb(b, pts, d, s, z, nullptr, P);      // B = beta2 + MB2 + s delta2
    g16_store(b_out, b, P);
}

}  // namespace cw

#if defined(__CUDACC__) && defined(CW_GROTH16_KERNELS)
// ---- kernel (sm_90a) --------------------------------------------------------------------------------------------------
namespace cw {

constexpr u32 G16_THREADS = 64;

// proofs [count][64] u32 = A (x, y) | B (x.c0, x.c1, y.c0, y.c1) | C (x, y), canonical.  ma, mb1, mc, mh: [count][16] u32,
// mb2: [count][32] u32, rs: [count][2][8] u32 (r, s), all canonical.  grid = (ceil(count / G16_THREADS), 2).
__global__ void __launch_bounds__(G16_THREADS) groth16_assemble_kernel(const Groth16Consts *__restrict__ K,
                                                                       const u32 *__restrict__ ma, const u32 *__restrict__ mb1,
                                                                       const u32 *__restrict__ mb2, const u32 *__restrict__ mc,
                                                                       const u32 *__restrict__ mh, const u32 *__restrict__ rs,
                                                                       u32 count, u32 *__restrict__ proofs) {
    const FrParams &P = c_fr[MSM_PRIME];
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    u32 out[32];
    u32 *pf = proofs + 64 * (size_t)i;
    if (blockIdx.y == 0) {
        groth16_g1(out, out + 16, *K, ma + 16 * (size_t)i, mb1 + 16 * (size_t)i, mc + 16 * (size_t)i, mh + 16 * (size_t)i,
                   rs + 16 * (size_t)i, rs + 16 * (size_t)i + 8, P);
        for (int k = 0; k < 16; k += 8) stg256(pf + k, out + k);
        for (int k = 0; k < 16; k += 8) stg256(pf + 48 + k, out + 16 + k);
    } else {
        groth16_g2(out, *K, mb2 + 32 * (size_t)i, rs + 16 * (size_t)i + 8, P);
        for (int k = 0; k < 32; k += 8) stg256(pf + 16 + k, out + k);
    }
}

}  // namespace cw
#endif
