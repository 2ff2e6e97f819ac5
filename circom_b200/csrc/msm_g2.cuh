// Multi-scalar multiplication on G2 of BN254: the twist E': y^2 = x^3 + b' over Fq2 = Fq[u] / (u^2 + 1), b' = 3 / (9 + u),
// q the base field of G1 (MSM_PRIME).  Same pipeline as msm.cuh - signed digits, the sort of keys, the run levels, the
// segment / window / Horner reduction - over a larger point type: the run and reduction functions of msm.cuh are
// templates over the bucket type and find the G2 point functions below by overloading.  Host and device, like msm.cuh;
// tests/hostsim/msm_g2_sim.cpp runs whole G2 MSMs on the CPU through these functions.
//
// An Fq2 element c0 + c1 u is two Montgomery images mod q.  Buckets are XYZZ over Fq2 (XyzzG2, 256 bytes), infinity is
// ZZ = 0, so zeroed memory is a row of empty buckets.  #E'(Fq2) = r (2q - r) is odd, so no point of E' has y = 0 and the
// exceptional cases of msm.cuh's formulas (equal points double, opposite points cancel) are the only ones, also for points
// outside the order-r subgroup.  Affine bases are [x.c0, x.c1, y.c0, y.c1] with all zeros for infinity (not on E': b' != 0).
#pragma once
#include "msm.cuh"

namespace cw {

// ---- Fq2 ---------------------------------------------------------------------------------------------------------------
struct alignas(16) Fq2 {
    u32 c0[8], c1[8];
};

CW_HD void fq2_set(Fq2 &r, const Fq2 &a) { u256_set(r.c0, a.c0); u256_set(r.c1, a.c1); }
CW_HD void fq2_zero(Fq2 &r) { u256_set_u32(r.c0, 0); u256_set_u32(r.c1, 0); }
CW_HD bool fq2_is_zero(const Fq2 &a) { return u256_is_zero(a.c0) && u256_is_zero(a.c1); }
CW_HD void fq2_add(Fq2 &r, const Fq2 &a, const Fq2 &b, const FrParams &P) {
    fr_add(r.c0, a.c0, b.c0, P);
    fr_add(r.c1, a.c1, b.c1, P);
}
CW_HD void fq2_sub(Fq2 &r, const Fq2 &a, const Fq2 &b, const FrParams &P) {
    fr_sub(r.c0, a.c0, b.c0, P);
    fr_sub(r.c1, a.c1, b.c1, P);
}
CW_HD void fq2_neg(Fq2 &r, const Fq2 &a, const FrParams &P) {
    fr_neg(r.c0, a.c0, P);
    fr_neg(r.c1, a.c1, P);
}
// Karatsuba, 3 products: (a0 b0 - a1 b1) + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) u.  r may be a or b.
CW_HD void fq2_mul(Fq2 &r, const Fq2 &a, const Fq2 &b, const FrParams &P) {
    u32 t0[8], t1[8], s[8], v[8];
    fr_mont_mul(t0, a.c0, b.c0, P);
    fr_mont_mul(t1, a.c1, b.c1, P);
    fr_add(s, a.c0, a.c1, P);
    fr_add(v, b.c0, b.c1, P);
    fr_mont_mul(s, s, v, P);
    fr_sub(r.c0, t0, t1, P);
    fr_sub(s, s, t0, P);
    fr_sub(r.c1, s, t1, P);
}
// 2 products: (a0 + a1)(a0 - a1) + 2 a0 a1 u.  r may be a.
CW_HD void fq2_sqr(Fq2 &r, const Fq2 &a, const FrParams &P) {
    u32 s[8], d[8], m[8];
    fr_add(s, a.c0, a.c1, P);
    fr_sub(d, a.c0, a.c1, P);
    fr_mont_mul(m, a.c0, a.c1, P);
    fr_mont_mul(r.c0, s, d, P);
    fr_add(r.c1, m, m, P);
}
// conj(a) / (a0^2 + a1^2): one inversion in Fq; zero maps to zero
CW_HD void fq2_inv(Fq2 &r, const Fq2 &a, const FrParams &P) {
    u32 n[8], t[8], inv[8];
    fr_mont_mul(n, a.c0, a.c0, P);
    fr_mont_mul(t, a.c1, a.c1, P);
    fr_add(n, n, t, P);
    fr_inv_mont(inv, n, P);
    fr_mont_mul(r.c0, a.c0, inv, P);
    fr_mont_mul(t, a.c1, inv, P);
    fr_neg(r.c1, t, P);
}

// ---- XYZZ points over Fq2 ----------------------------------------------------------------------------------------------
struct alignas(16) XyzzG2 {
    Fq2 x, y, zz, zzz;
};

CW_HD void xyzz_inf(XyzzG2 &p) { fq2_zero(p.x); fq2_zero(p.y); fq2_zero(p.zz); fq2_zero(p.zzz); }
CW_HD bool xyzz_is_inf(const XyzzG2 &p) { return fq2_is_zero(p.zz); }

// dbl-2008-s-1 (a = 0), as xyzz_dbl of msm.cuh; infinity stays infinity (ZZ = 0)
CW_HD void xyzz_dbl(XyzzG2 &p, const FrParams &P) {
    Fq2 u, v, w, s, m, t;
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
CW_HD void xyzz_madd(XyzzG2 &a, const Fq2 &x2, const Fq2 &y2, const FrParams &P) {
    if (fq2_is_zero(x2) && fq2_is_zero(y2)) return;
    if (xyzz_is_inf(a)) {
        fq2_set(a.x, x2); fq2_set(a.y, y2);
        u256_set(a.zz.c0, P.r1); u256_set_u32(a.zz.c1, 0);
        u256_set(a.zzz.c0, P.r1); u256_set_u32(a.zzz.c1, 0);
        return;
    }
    Fq2 pp, r, ppp, q, t;
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
CW_HD void xyzz_add(XyzzG2 &a, const XyzzG2 &b, const FrParams &P) {
    if (xyzz_is_inf(b)) return;
    if (xyzz_is_inf(a)) {
        a = b;
        return;
    }
    Fq2 u1, s1, pp, r, ppp, q, t;
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
CW_HD void xyzz_to_affine(Fq2 &x, Fq2 &y, const XyzzG2 &p, const FrParams &P) {
    if (xyzz_is_inf(p)) {
        fq2_zero(x);
        fq2_zero(y);
        return;
    }
    Fq2 t, inv;
    fq2_mul(t, p.zz, p.zzz, P);
    fq2_inv(inv, t, P);                 // 1 / (ZZ ZZZ)
    fq2_mul(t, inv, p.zzz, P);          // 1 / ZZ
    fq2_mul(x, p.x, t, P);
    fq2_mul(t, inv, p.zz, P);           // 1 / ZZZ
    fq2_mul(y, p.y, t, P);
}

CW_HD void msm_ld_fq2(Fq2 &a, const u32 *s) {
    ntt_ld8(a.c0, s);
    ntt_ld8(a.c1, s + 8);
}
CW_HD void msm_ld_xyzz(XyzzG2 &p, const XyzzG2 *src) {
    const u32 *s = (const u32 *)src;
    msm_ld_fq2(p.x, s);
    msm_ld_fq2(p.y, s + 16);
    msm_ld_fq2(p.zz, s + 32);
    msm_ld_fq2(p.zzz, s + 48);
}

// the items of the first level: sorted (key, point index | sign << 31) over the affine bases [n][32] u32 (Montgomery
// x.c0, x.c1, y.c0, y.c1)
struct MsmG2AffineItems {
    const u32 *keys, *vals, *bases;
    CW_HD void add(XyzzG2 &acc, uint64_t i, const FrParams &P) const {
        const u32 v = vals[i];
        Fq2 x, y;
        const u32 *b = bases + 32 * (size_t)(v & 0x7FFFFFFFu);
        msm_ld_fq2(x, b);
        msm_ld_fq2(y, b + 16);
        if (v >> 31) fq2_neg(y, y, P);
        xyzz_madd(acc, x, y, P);
    }
};
// the items of the later levels: partial sums left by the level before
struct MsmG2XyzzItems {
    const u32 *keys;
    const XyzzG2 *pts;
    CW_HD void add(XyzzG2 &acc, uint64_t i, const FrParams &P) const {
        XyzzG2 p;
        msm_ld_xyzz(p, pts + i);
        xyzz_add(acc, p, P);
    }
};

}  // namespace cw

#if defined(__CUDACC__) && !defined(CW_MSM_NO_G2_KERNELS)   // (groth16.cu uses the point functions only)
// ---- kernels (sm_90a) -------------------------------------------------------------------------------------------------
// The digits and the sort are msm.cuh's (they do not depend on the group).  The bucket type is four times the G1 one, so
// the kernels run MSM_G2_THREADS threads per CTA, which lets ptxas use up to 255 registers per thread (DESIGN section 4).
namespace cw {

constexpr u32 MSM_G2_THREADS = 128;

template <bool AFFINE>
__global__ void __launch_bounds__(MSM_G2_THREADS) msm_g2_runs_kernel(const u32 *__restrict__ keys, const u32 *__restrict__ vals,
                                                                     const u32 *__restrict__ bases,
                                                                     const XyzzG2 *__restrict__ pts, uint64_t N, u32 c,
                                                                     XyzzG2 *buckets, u32 *okeys, XyzzG2 *opts) {
    const FrParams &P = c_fr[MSM_PRIME];
    const uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= threads) return;
    MsmRunOutT<XyzzG2> o{buckets, okeys, opts};
    if (AFFINE) msm_sum_runs(MsmG2AffineItems{keys, vals, bases}, N, t, c, o, P);
    else msm_sum_runs(MsmG2XyzzItems{keys, pts}, N, t, c, o, P);
}

// segment results: thread per (window of the chunk, segment of MSM_SEG buckets)
__global__ void __launch_bounds__(MSM_G2_THREADS) msm_g2_segments_kernel(const XyzzG2 *__restrict__ buckets, u32 B, u32 n_win,
                                                                         XyzzG2 *__restrict__ segs) {
    const FrParams &P = c_fr[MSM_PRIME];
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n_win * per) return;
    const u32 w = (u32)(t / per), s = (u32)(t % per);
    XyzzG2 r;
    msm_bucket_segment(r, buckets + (size_t)w * B, s * m, m, P);
    segs[t] = r;
}

// window sums: one CTA per window of the chunk adds its `per` segment results
__global__ void __launch_bounds__(MSM_G2_THREADS) msm_g2_windows_kernel(const XyzzG2 *__restrict__ segs, u32 per,
                                                                        XyzzG2 *__restrict__ wins) {
    __shared__ XyzzG2 sm[MSM_G2_THREADS];
    const FrParams &P = c_fr[MSM_PRIME];
    XyzzG2 acc, b;
    xyzz_inf(acc);
    for (u32 s = threadIdx.x; s < per; s += MSM_G2_THREADS) {
        msm_ld_xyzz(b, segs + (size_t)blockIdx.x * per + s);
        xyzz_add(acc, b, P);
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (u32 h = MSM_G2_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            acc = sm[threadIdx.x];
            xyzz_add(acc, sm[threadIdx.x + h], P);
            sm[threadIdx.x] = acc;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) wins[blockIdx.x] = sm[0];
}

// one thread per instance: Horner's rule over its W window sums, then affine canonical [2][2][4] u64
__global__ void __launch_bounds__(MSM_G2_THREADS) msm_g2_final_kernel(const XyzzG2 *__restrict__ wins, u32 W, u32 c, u32 count,
                                                                      uint4 *__restrict__ out) {
    const FrParams &P = c_fr[MSM_PRIME];
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    XyzzG2 acc;
    msm_horner(acc, wins + (size_t)i * W, W, c, P);
    Fq2 x, y;
    xyzz_to_affine(x, y, acc, P);
    u32 v[8];
    uint4 *o = out + 8 * (size_t)i;
    fr_from_mont(v, x.c0, P);
    stg256(o, v);
    fr_from_mont(v, x.c1, P);
    stg256(o + 2, v);
    fr_from_mont(v, y.c0, P);
    stg256(o + 4, v);
    fr_from_mont(v, y.c1, P);
    stg256(o + 6, v);
}

}  // namespace cw
#endif
