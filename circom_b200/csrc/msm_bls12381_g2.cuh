// Multi-scalar multiplication on G2 of BLS12-381: the twist E': y^2 = x^3 + 4 (1 + u) over Fq2 = Fq[u] / (u^2 + 1), q the
// 381-bit base field of BLS12-381 G1 (msm_bls12381.cuh), group order r (the library's bls12381 prime), cofactor
// h2 = 0x5d543a95...1c7238e5 (507 bits, odd).  The same pipeline as msm.cuh - signed digits, the sort of keys, the run
// levels, the segment / window / Horner reduction - over the largest point type of the library: the run and reduction
// functions of msm.cuh are templates over the bucket type and the parameter record, and find the point functions below by
// overloading.  Host and device, like msm.cuh; tests/hostsim/msm_bls12381_g2_sim.cpp runs the field, the formulas and
// whole MSMs on the CPU through these functions.
//
// An Fq2 element c0 + c1 u is two 12-limb Montgomery images mod q (Fq2_381, 96 bytes); q = 3 mod 4, so -1 is the
// non-residue, as for BN254's Fq2, and the product, square and inverse are msm_g2.cuh's.  Buckets are XYZZ over Fq2
// (XyzzG2_381, 384 bytes), infinity is ZZ = 0, so zeroed memory is a row of empty buckets.  #E'(Fq2) = h2 r is odd, so no
// point of E' has y = 0 and the exceptional cases of the formulas (equal points double, opposite points cancel) are the
// only ones, also for points outside the order-r subgroup.  Affine bases are [x.c0, x.c1, y.c0, y.c1] (48 u32) with all
// zeros for infinity (not on E': b' != 0).
//
// The Fq2 product, square and inverse are out-of-line functions on the device (FQ2_381_FN): a full XYZZ addition is 40
// twelve-limb products, and with every one of them inlined into every use the unit would take the device compiler many
// times longer than the other MSM units.  Out of line, each product is compiled once per unit, and the point formulas
// around them stay small.  DESIGN section 7 measures what the calls cost.
#pragma once
#include "msm_bls12381.cuh"

#if defined(__CUDACC__)
#define FQ2_381_FN __host__ __device__ __noinline__
#else
#define FQ2_381_FN inline
#endif

namespace cw {

// b' = 4 (1 + u) of y^2 = x^3 + b', canonical (c0, c1)
constexpr u32 BLS12381_G2_B0 = 4, BLS12381_G2_B1 = 4;

// ---- Fq2 over the 12-limb field -----------------------------------------------------------------------------------------
struct alignas(16) Fq2_381 {
    u32 c0[12], c1[12];
};

CW_HD void fq2_set(Fq2_381 &r, const Fq2_381 &a) { fp381_set(r.c0, a.c0); fp381_set(r.c1, a.c1); }
CW_HD void fq2_zero(Fq2_381 &r) { fp381_set_u32(r.c0, 0); fp381_set_u32(r.c1, 0); }
CW_HD bool fq2_is_zero(const Fq2_381 &a) { return fp381_is_zero(a.c0) && fp381_is_zero(a.c1); }
CW_HD void fq2_add(Fq2_381 &r, const Fq2_381 &a, const Fq2_381 &b, const Fp381Params &P) {
    fp381_add(r.c0, a.c0, b.c0, P);
    fp381_add(r.c1, a.c1, b.c1, P);
}
CW_HD void fq2_sub(Fq2_381 &r, const Fq2_381 &a, const Fq2_381 &b, const Fp381Params &P) {
    fp381_sub(r.c0, a.c0, b.c0, P);
    fp381_sub(r.c1, a.c1, b.c1, P);
}
CW_HD void fq2_neg(Fq2_381 &r, const Fq2_381 &a, const Fp381Params &P) {
    fp381_neg(r.c0, a.c0, P);
    fp381_neg(r.c1, a.c1, P);
}
// Karatsuba, 3 products: (a0 b0 - a1 b1) + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) u.  r may be a or b.
FQ2_381_FN void fq2_mul(Fq2_381 &r, const Fq2_381 &a, const Fq2_381 &b, const Fp381Params &P) {
    u32 t0[12], t1[12], s[12], v[12];
    fp381_mul(t0, a.c0, b.c0, P);
    fp381_mul(t1, a.c1, b.c1, P);
    fp381_add(s, a.c0, a.c1, P);
    fp381_add(v, b.c0, b.c1, P);
    fp381_mul(s, s, v, P);
    fp381_sub(r.c0, t0, t1, P);
    fp381_sub(s, s, t0, P);
    fp381_sub(r.c1, s, t1, P);
}
// 2 products: (a0 + a1)(a0 - a1) + 2 a0 a1 u.  r may be a.
FQ2_381_FN void fq2_sqr(Fq2_381 &r, const Fq2_381 &a, const Fp381Params &P) {
    u32 s[12], d[12], m[12];
    fp381_add(s, a.c0, a.c1, P);
    fp381_sub(d, a.c0, a.c1, P);
    fp381_mul(m, a.c0, a.c1, P);
    fp381_mul(r.c0, s, d, P);
    fp381_add(r.c1, m, m, P);
}
// conj(a) / (a0^2 + a1^2): one inversion in Fq; zero maps to zero
FQ2_381_FN void fq2_inv(Fq2_381 &r, const Fq2_381 &a, const Fp381Params &P) {
    u32 n[12], t[12], inv[12];
    fp381_mul(n, a.c0, a.c0, P);
    fp381_mul(t, a.c1, a.c1, P);
    fp381_add(n, n, t, P);
    fp381_inv(inv, n, P);
    fp381_mul(r.c0, a.c0, inv, P);
    fp381_mul(t, a.c1, inv, P);
    fp381_neg(r.c1, t, P);
}

// ---- XYZZ points over Fq2 ----------------------------------------------------------------------------------------------
struct alignas(16) XyzzG2_381 {
    Fq2_381 x, y, zz, zzz;
};

CW_HD void xyzz_inf(XyzzG2_381 &p) { fq2_zero(p.x); fq2_zero(p.y); fq2_zero(p.zz); fq2_zero(p.zzz); }
CW_HD bool xyzz_is_inf(const XyzzG2_381 &p) { return fq2_is_zero(p.zz); }

// dbl-2008-s-1 (a = 0), as xyzz_dbl of msm_g2.cuh; infinity stays infinity (ZZ = 0)
CW_HD void xyzz_dbl(XyzzG2_381 &p, const Fp381Params &P) {
    Fq2_381 u, v, w, s, m, t;
    fq2_add(u, p.y, p.y, P);
    fq2_sqr(v, u, P);
    fq2_mul(w, u, v, P);
    fq2_mul(s, p.x, v, P);
    fq2_sqr(t, p.x, P);
    fq2_add(m, t, t, P);
    fq2_add(m, m, t, P);                // M = 3 X^2
    fq2_sqr(t, m, P);
    fq2_sub(t, t, s, P);
    fq2_sub(p.x, t, s, P);              // X3 = M^2 - 2 S
    fq2_sub(t, s, p.x, P);
    fq2_mul(s, m, t, P);
    fq2_mul(t, w, p.y, P);
    fq2_sub(p.y, s, t, P);              // Y3 = M (S - X3) - W Y1
    fq2_mul(p.zz, v, p.zz, P);
    fq2_mul(p.zzz, w, p.zzz, P);
}

// acc += (x2, y2) affine, madd-2008-s.  Equal points double, opposite points give infinity; all-zero (x2, y2) is infinity.
CW_HD void xyzz_madd(XyzzG2_381 &a, const Fq2_381 &x2, const Fq2_381 &y2, const Fp381Params &P) {
    if (fq2_is_zero(x2) && fq2_is_zero(y2)) return;
    if (xyzz_is_inf(a)) {
        fq2_set(a.x, x2); fq2_set(a.y, y2);
        fp381_set(a.zz.c0, P.r1); fp381_set_u32(a.zz.c1, 0);
        fp381_set(a.zzz.c0, P.r1); fp381_set_u32(a.zzz.c1, 0);
        return;
    }
    Fq2_381 pp, r, ppp, q, t;
    fq2_mul(t, x2, a.zz, P);
    fq2_sub(pp, t, a.x, P);             // P = U2 - X1
    fq2_mul(t, y2, a.zzz, P);
    fq2_sub(r, t, a.y, P);              // R = S2 - Y1
    if (fq2_is_zero(pp)) {
        if (fq2_is_zero(r)) xyzz_dbl(a, P);
        else xyzz_inf(a);
        return;
    }
    fq2_sqr(t, pp, P);
    fq2_mul(ppp, pp, t, P);             // PPP = P^3
    fq2_mul(q, a.x, t, P);              // Q = X1 PP
    fq2_mul(a.zz, a.zz, t, P);          // ZZ3 = ZZ1 PP
    fq2_mul(a.zzz, a.zzz, ppp, P);      // ZZZ3 = ZZZ1 PPP
    fq2_sqr(t, r, P);
    fq2_sub(t, t, ppp, P);
    fq2_sub(t, t, q, P);
    fq2_sub(a.x, t, q, P);              // X3 = R^2 - PPP - 2 Q
    fq2_sub(t, q, a.x, P);
    fq2_mul(q, r, t, P);
    fq2_mul(t, a.y, ppp, P);
    fq2_sub(a.y, q, t, P);              // Y3 = R (Q - X3) - Y1 PPP
}

// a += b, add-2008-s, with the same exceptional cases
CW_HD void xyzz_add(XyzzG2_381 &a, const XyzzG2_381 &b, const Fp381Params &P) {
    if (xyzz_is_inf(b)) return;
    if (xyzz_is_inf(a)) {
        a = b;
        return;
    }
    Fq2_381 u1, s1, pp, r, ppp, q, t;
    fq2_mul(u1, a.x, b.zz, P);
    fq2_mul(t, b.x, a.zz, P);
    fq2_sub(pp, t, u1, P);              // P = U2 - U1
    fq2_mul(s1, a.y, b.zzz, P);
    fq2_mul(t, b.y, a.zzz, P);
    fq2_sub(r, t, s1, P);               // R = S2 - S1
    if (fq2_is_zero(pp)) {
        if (fq2_is_zero(r)) xyzz_dbl(a, P);
        else xyzz_inf(a);
        return;
    }
    fq2_sqr(t, pp, P);
    fq2_mul(ppp, pp, t, P);
    fq2_mul(q, u1, t, P);
    fq2_mul(a.zz, a.zz, b.zz, P);
    fq2_mul(a.zz, a.zz, t, P);          // ZZ3 = ZZ1 ZZ2 PP
    fq2_mul(a.zzz, a.zzz, b.zzz, P);
    fq2_mul(a.zzz, a.zzz, ppp, P);      // ZZZ3 = ZZZ1 ZZZ2 PPP
    fq2_sqr(t, r, P);
    fq2_sub(t, t, ppp, P);
    fq2_sub(t, t, q, P);
    fq2_sub(a.x, t, q, P);
    fq2_sub(t, q, a.x, P);
    fq2_mul(q, r, t, P);
    fq2_mul(t, s1, ppp, P);
    fq2_sub(a.y, q, t, P);              // Y3 = R (Q - X3) - S1 PPP
}

// affine Montgomery coordinates of p, all zeros for infinity: one Fq2 inversion of ZZ ZZZ
CW_HD void xyzz_to_affine(Fq2_381 &x, Fq2_381 &y, const XyzzG2_381 &p, const Fp381Params &P) {
    if (xyzz_is_inf(p)) {
        fq2_zero(x);
        fq2_zero(y);
        return;
    }
    Fq2_381 t, inv;
    fq2_mul(t, p.zz, p.zzz, P);
    fq2_inv(inv, t, P);                 // 1 / (ZZ ZZZ)
    fq2_mul(t, inv, p.zzz, P);          // 1 / ZZ
    fq2_mul(x, p.x, t, P);
    fq2_mul(t, inv, p.zz, P);           // 1 / ZZZ
    fq2_mul(y, p.y, t, P);
}

CW_HD void msm_ld_fq2(Fq2_381 &a, const u32 *s) {
    fp381_ld(a.c0, s);
    fp381_ld(a.c1, s + 12);
}
CW_HD void msm_ld_xyzz(XyzzG2_381 &p, const XyzzG2_381 *src) {
    const u32 *s = (const u32 *)src;
    msm_ld_fq2(p.x, s);
    msm_ld_fq2(p.y, s + 24);
    msm_ld_fq2(p.zz, s + 48);
    msm_ld_fq2(p.zzz, s + 72);
}

// canonical affine (x.c0, x.c1, y.c0, y.c1), 12 limbs each, to Montgomery images in mont[48]: 0 on E' or all zeros, 1 a
// coefficient not below q (*bad its index 0..3), 2 not on the twist (the host checks of the ABI)
CW_HD int bls12381_g2_to_mont(u32 *mont, const u32 *canon, int *bad, const Fp381Params &P) {
    bool zero = true;
    for (int k = 0; k < 4; ++k) zero = zero && fp381_is_zero(canon + 12 * k);
    if (zero) {
        for (int k = 0; k < 48; ++k) mont[k] = 0;
        return 0;
    }
    for (int k = 0; k < 4; ++k)
        if (!fp381_lt_q(canon + 12 * k, P)) {
            *bad = k;
            return 1;
        }
    Fq2_381 x, y, b, lhs, rhs;
    fp381_to_mont(x.c0, canon, P);
    fp381_to_mont(x.c1, canon + 12, P);
    fp381_to_mont(y.c0, canon + 24, P);
    fp381_to_mont(y.c1, canon + 36, P);
    fp381_set_u32(b.c0, BLS12381_G2_B0);
    fp381_set_u32(b.c1, BLS12381_G2_B1);
    fp381_to_mont(b.c0, b.c0, P);
    fp381_to_mont(b.c1, b.c1, P);
    fq2_sqr(lhs, y, P);
    fq2_sqr(rhs, x, P);
    fq2_mul(rhs, rhs, x, P);
    fq2_add(rhs, rhs, b, P);
    fp381_set(mont, x.c0);
    fp381_set(mont + 12, x.c1);
    fp381_set(mont + 24, y.c0);
    fp381_set(mont + 36, y.c1);
    return fp381_eq(lhs.c0, rhs.c0) && fp381_eq(lhs.c1, rhs.c1) ? 0 : 2;
}

// the items of the first level: sorted (key, point index | sign << 31) over the affine bases [n][48] u32 (Montgomery
// x.c0, x.c1, y.c0, y.c1)
struct MsmBlsG2AffineItems {
    const u32 *keys, *vals, *bases;
    CW_HD void add(XyzzG2_381 &acc, uint64_t i, const Fp381Params &P) const {
        const u32 v = vals[i];
        Fq2_381 x, y;
        const u32 *b = bases + 48 * (size_t)(v & 0x7FFFFFFFu);
        msm_ld_fq2(x, b);
        msm_ld_fq2(y, b + 24);
        if (v >> 31) fq2_neg(y, y, P);
        xyzz_madd(acc, x, y, P);
    }
};
// the items of the later levels: partial sums left by the level before
struct MsmBlsG2XyzzItems {
    const u32 *keys;
    const XyzzG2_381 *pts;
    CW_HD void add(XyzzG2_381 &acc, uint64_t i, const Fp381Params &P) const {
        XyzzG2_381 p;
        msm_ld_xyzz(p, pts + i);
        xyzz_add(acc, p, P);
    }
};

}  // namespace cw

#if defined(__CUDACC__)
// ---- kernels (sm_90a) -------------------------------------------------------------------------------------------------
// The digits and the sort are msm.cuh's (they do not depend on the group).  The run, segment and final kernels run
// MSM_BLS_G2_THREADS threads per CTA, which lets ptxas use up to 255 registers per thread (DESIGN section 4).  The
// windows kernel keeps one point per thread in shared memory: at 384 bytes a point, MSM_BLS_G2_WIN_THREADS = 64 threads
// take 24 KB, half the static limit.
namespace cw {

constexpr u32 MSM_BLS_G2_THREADS = 128;
constexpr u32 MSM_BLS_G2_WIN_THREADS = 64;

__constant__ Fp381Params c_fp381_g2;

template <bool AFFINE>
__global__ void __launch_bounds__(MSM_BLS_G2_THREADS) msm_bls_g2_runs_kernel(const u32 *__restrict__ keys,
                                                                             const u32 *__restrict__ vals,
                                                                             const u32 *__restrict__ bases,
                                                                             const XyzzG2_381 *__restrict__ pts, uint64_t N,
                                                                             u32 c, XyzzG2_381 *buckets, u32 *okeys,
                                                                             XyzzG2_381 *opts) {
    const Fp381Params &P = c_fp381_g2;
    const uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= threads) return;
    MsmRunOutT<XyzzG2_381> o{buckets, okeys, opts};
    if (AFFINE) msm_sum_runs(MsmBlsG2AffineItems{keys, vals, bases}, N, t, c, o, P);
    else msm_sum_runs(MsmBlsG2XyzzItems{keys, pts}, N, t, c, o, P);
}

// segment results: thread per (window of the chunk, segment of MSM_SEG buckets)
__global__ void __launch_bounds__(MSM_BLS_G2_THREADS) msm_bls_g2_segments_kernel(const XyzzG2_381 *__restrict__ buckets, u32 B,
                                                                                 u32 n_win, XyzzG2_381 *__restrict__ segs) {
    const Fp381Params &P = c_fp381_g2;
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n_win * per) return;
    const u32 w = (u32)(t / per), s = (u32)(t % per);
    XyzzG2_381 r;
    msm_bucket_segment(r, buckets + (size_t)w * B, s * m, m, P);
    segs[t] = r;
}

// window sums: one CTA per window of the chunk adds its `per` segment results
__global__ void __launch_bounds__(MSM_BLS_G2_WIN_THREADS) msm_bls_g2_windows_kernel(const XyzzG2_381 *__restrict__ segs, u32 per,
                                                                                    XyzzG2_381 *__restrict__ wins) {
    __shared__ XyzzG2_381 sm[MSM_BLS_G2_WIN_THREADS];
    const Fp381Params &P = c_fp381_g2;
    XyzzG2_381 acc, b;
    xyzz_inf(acc);
    for (u32 s = threadIdx.x; s < per; s += MSM_BLS_G2_WIN_THREADS) {
        msm_ld_xyzz(b, segs + (size_t)blockIdx.x * per + s);
        xyzz_add(acc, b, P);
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (u32 h = MSM_BLS_G2_WIN_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            acc = sm[threadIdx.x];
            xyzz_add(acc, sm[threadIdx.x + h], P);
            sm[threadIdx.x] = acc;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) wins[blockIdx.x] = sm[0];
}

// one thread per instance: Horner's rule over its W window sums as one flat loop (as msm_bls_final_kernel runs it), then
// affine canonical [2][2][6] u64
__global__ void __launch_bounds__(MSM_BLS_G2_THREADS) msm_bls_g2_final_kernel(const XyzzG2_381 *__restrict__ wins, u32 W, u32 c,
                                                                              u32 count, uint4 *__restrict__ out) {
    const Fp381Params &P = c_fp381_g2;
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const XyzzG2_381 *win = wins + (size_t)i * W;
    XyzzG2_381 acc, s;
    msm_ld_xyzz(acc, win + (W - 1));
    u32 w = W - 1, k = 0;
#pragma unroll 1
    while (w > 0) {
        if (k < c) {
            xyzz_dbl(acc, P);
            ++k;
        } else {
            msm_ld_xyzz(s, win + --w);
            xyzz_add(acc, s, P);
            k = 0;
        }
    }
    Fq2_381 x, y;
    xyzz_to_affine(x, y, acc, P);
    uint4 *o = out + 12 * (size_t)i;
    const u32 *coef[4] = {x.c0, x.c1, y.c0, y.c1};
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
        u32 v[12];
        fp381_from_mont(v, coef[j], P);
        for (int k = 0; k < 3; ++k) o[3 * j + k] = make_uint4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
    }
}

}  // namespace cw
#endif
