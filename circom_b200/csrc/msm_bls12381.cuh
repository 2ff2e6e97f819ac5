// Multi-scalar multiplication on G1 of BLS12-381: y^2 = x^3 + 4 over the 381-bit base field q, group order r (the
// library's bls12381 prime, 255 bits), cofactor h = 0x396c8c005555e1568c00aaab0000aaab.  The same pipeline as msm.cuh -
// signed digits, the sort of keys, the run levels, the segment / window / Horner reduction - over a wider field: the run
// and reduction functions of msm.cuh are templates over the bucket type and the parameter record, and find the point
// functions below by overloading.  Host and device, like msm.cuh; tests/hostsim/msm_bls12381_sim.cpp runs the field, the
// formulas and whole MSMs on the CPU through these functions.
//
// The field: 12 x u32 limbs, little-endian, Montgomery images with R = 2^384.  q < 2^381, so sums of two reduced values
// and the CIOS product's result (< 2q) fit 12 limbs.  The 8-limb functions of fr_device.cuh are not touched: this is a
// separate set with its own parameter record (Fp381Params).
//
// Buckets are XYZZ over Fq (Xyzz381, 192 bytes), infinity is ZZ = 0, so zeroed memory is a row of empty buckets.  h and r
// are odd, so #E(Fq) = h r is odd and no point has y = 0: the exceptional cases of the formulas are equal points (they
// double) and opposite points (they cancel), also for points outside the order-r subgroup.  Affine bases are [n][24] u32
// Montgomery (x, y) with (0, 0) for infinity (not on the curve: 4 != 0).
#pragma once
#include "msm.cuh"

namespace cw {

struct Fp381Params {
    u32 q[12];     // modulus
    u32 r1[12];    // 2^384 mod q: Montgomery image of 1
    u32 r2[12];    // 2^768 mod q
    u32 qm2[12];   // q - 2 (Fermat exponent)
    u32 np32;      // -q^-1 mod 2^32
    u32 pad[3];
};

// the constants of BLS12-381's base field (checked against Python integers by tests/test_bls12381_msm_cpu.py)
inline Fp381Params fp381_params() {
    return Fp381Params{
        {0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u,
         0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau},
        {0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu, 0x53c758bau, 0x5f489857u, 0x70525745u, 0x77ce5853u,
         0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u},
        {0x1c341746u, 0xf4df1f34u, 0x09d104f1u, 0x0a76e6a6u, 0x4c95b6d5u, 0x8de5476cu, 0x939d83c0u, 0x67eb88a9u,
         0xb519952du, 0x9a793e85u, 0x92cae3aau, 0x11988fe5u},
        {0xffffaaa9u, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u,
         0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau},
        0xfffcfffdu,
        {0, 0, 0}};
}

// b = 4 of y^2 = x^3 + b, canonical
constexpr u32 BLS12381_B = 4;

// ---- Fq, 12 limbs --------------------------------------------------------------------------------------------------------
CW_HD void fp381_set(u32 *r, const u32 *a) {
#pragma unroll
    for (int i = 0; i < 12; ++i) r[i] = a[i];
}
CW_HD void fp381_set_u32(u32 *r, u32 v) {
    r[0] = v;
#pragma unroll
    for (int i = 1; i < 12; ++i) r[i] = 0;
}
CW_HD bool fp381_is_zero(const u32 *a) {
    u32 o = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) o |= a[i];
    return o == 0;
}
CW_HD bool fp381_eq(const u32 *a, const u32 *b) {
    u32 o = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) o |= a[i] ^ b[i];
    return o == 0;
}
// r = a - b over 12 limbs; returns the borrow (0 / 1)
CW_HD u32 fp381_sub_raw(u32 *r, const u32 *a, const u32 *b) {
    u32 br = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
        const u64 t = (u64)a[i] - b[i] - br;
        r[i] = (u32)t;
        br = (u32)(t >> 63);
    }
    return br;
}
// a < q for a canonical value (the host checks of the ABI)
CW_HD bool fp381_lt_q(const u32 *a, const Fp381Params &P) {
    u32 t[12];
    return fp381_sub_raw(t, a, P.q) != 0;
}
// a + b < 2q < 2^382: no carry out of the 12 limbs; one conditional subtraction
CW_HD void fp381_add(u32 *r, const u32 *a, const u32 *b, const Fp381Params &P) {
    u32 s[12], t[12];
    u64 c = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
        c += (u64)a[i] + b[i];
        s[i] = (u32)c;
        c >>= 32;
    }
    const u32 br = fp381_sub_raw(t, s, P.q);
#pragma unroll
    for (int i = 0; i < 12; ++i) r[i] = br ? s[i] : t[i];
}
CW_HD void fp381_sub(u32 *r, const u32 *a, const u32 *b, const Fp381Params &P) {
    u32 s[12], t[12];
    const u32 br = fp381_sub_raw(s, a, b);
    u64 c = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
        c += (u64)s[i] + P.q[i];
        t[i] = (u32)c;
        c >>= 32;
    }
#pragma unroll
    for (int i = 0; i < 12; ++i) r[i] = br ? t[i] : s[i];
}
CW_HD void fp381_neg(u32 *r, const u32 *a, const Fp381Params &P) {
    u32 t[12];
    fp381_sub_raw(t, P.q, a);
    const bool z = fp381_is_zero(a);
#pragma unroll
    for (int i = 0; i < 12; ++i) r[i] = z ? 0u : t[i];
}

// Montgomery product a b 2^-384 mod q, CIOS.  With a, b < q the accumulator stays below 2q < 2^382 after every outer
// step, so it fits 12 limbs between steps; the 13th limb of a step's partial sum (t + a b_i) is carried in t12.
CW_HD void fp381_mul(u32 *r, const u32 *a, const u32 *b, const Fp381Params &P) {
    u32 t[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) t[i] = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
        u64 c = 0;
        const u32 bi = b[i];
#pragma unroll
        for (int j = 0; j < 12; ++j) {
            c += (u64)a[j] * bi + t[j];
            t[j] = (u32)c;
            c >>= 32;
        }
        const u32 t12 = (u32)c;
        const u32 m = t[0] * P.np32;
        c = ((u64)m * P.q[0] + t[0]) >> 32;
#pragma unroll
        for (int j = 1; j < 12; ++j) {
            c += (u64)m * P.q[j] + t[j];
            t[j - 1] = (u32)c;
            c >>= 32;
        }
        t[11] = (u32)(c + t12);   // (t + a b_i + m q) / 2^32 < 2q: no carry beyond
    }
    u32 d[12];
    const u32 br = fp381_sub_raw(d, t, P.q);
#pragma unroll
    for (int i = 0; i < 12; ++i) r[i] = br ? t[i] : d[i];
}

CW_HD void fp381_to_mont(u32 *r, const u32 *a, const Fp381Params &P) { fp381_mul(r, a, P.r2, P); }
CW_HD void fp381_from_mont(u32 *r, const u32 *a, const Fp381Params &P) {
    u32 one[12];
    fp381_set_u32(one, 1);
    fp381_mul(r, a, one, P);
}

// 1 / a in the Montgomery domain (aR -> a^-1 R): Fermat's ladder a^(q-2), about 570 products; zero maps to zero.  Used
// once per instance, in the final kernel.
CW_HD void fp381_inv(u32 *r, const u32 *a, const Fp381Params &P) {
    u32 acc[12], t[12], e[12];
    fp381_set(acc, P.r1);
    fp381_set(e, P.qm2);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int i = 0; i < 384; ++i) {
        const u32 bit = e[11] >> 31;   // the exponent is shifted in registers: no dynamically indexed array
#pragma unroll
        for (int j = 11; j > 0; --j) e[j] = (e[j] << 1) | (e[j - 1] >> 31);
        e[0] <<= 1;
        fp381_mul(t, acc, acc, P);
        if (bit) fp381_mul(acc, t, a, P);
        else fp381_set(acc, t);
    }
    fp381_set(r, acc);
}

// 12 limbs from (device: read-only) memory, 16-byte aligned
CW_HD void fp381_ld(u32 *v, const u32 *p) {
#if defined(__CUDA_ARCH__)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint4 w = __ldg((const uint4 *)p + k);
        v[4 * k] = w.x; v[4 * k + 1] = w.y; v[4 * k + 2] = w.z; v[4 * k + 3] = w.w;
    }
#else
    memcpy(v, p, 48);
#endif
}

// ---- XYZZ points over Fq -----------------------------------------------------------------------------------------------
struct alignas(16) Xyzz381 {
    u32 x[12], y[12], zz[12], zzz[12];
};

CW_HD void xyzz_inf(Xyzz381 &p) { fp381_set_u32(p.x, 0); fp381_set_u32(p.y, 0); fp381_set_u32(p.zz, 0); fp381_set_u32(p.zzz, 0); }
CW_HD bool xyzz_is_inf(const Xyzz381 &p) { return fp381_is_zero(p.zz); }

// dbl-2008-s-1 (a = 0), as xyzz_dbl of msm.cuh; infinity stays infinity (ZZ = 0)
CW_HD void xyzz_dbl(Xyzz381 &p, const Fp381Params &P) {
    u32 u[12], v[12], w[12], s[12], m[12], t[12];
    fp381_add(u, p.y, p.y, P);
    fp381_mul(v, u, u, P);
    fp381_mul(w, u, v, P);
    fp381_mul(s, p.x, v, P);
    fp381_mul(t, p.x, p.x, P);
    fp381_add(m, t, t, P);
    fp381_add(m, m, t, P);              // M = 3 X^2
    fp381_mul(t, m, m, P);
    fp381_sub(t, t, s, P);
    fp381_sub(p.x, t, s, P);            // X3 = M^2 - 2 S
    fp381_sub(t, s, p.x, P);
    fp381_mul(s, m, t, P);
    fp381_mul(t, w, p.y, P);
    fp381_sub(p.y, s, t, P);            // Y3 = M (S - X3) - W Y1
    fp381_mul(t, v, p.zz, P);
    fp381_set(p.zz, t);
    fp381_mul(t, w, p.zzz, P);
    fp381_set(p.zzz, t);
}

// acc += (x2, y2) affine, madd-2008-s.  Equal points double, opposite points give infinity; (0, 0) is infinity.
CW_HD void xyzz_madd(Xyzz381 &a, const u32 *x2, const u32 *y2, const Fp381Params &P) {
    if (fp381_is_zero(x2) && fp381_is_zero(y2)) return;
    if (xyzz_is_inf(a)) {
        fp381_set(a.x, x2); fp381_set(a.y, y2); fp381_set(a.zz, P.r1); fp381_set(a.zzz, P.r1);
        return;
    }
    u32 pp[12], r[12], ppp[12], q[12], t[12];
    fp381_mul(t, x2, a.zz, P);
    fp381_sub(pp, t, a.x, P);           // P = U2 - X1
    fp381_mul(t, y2, a.zzz, P);
    fp381_sub(r, t, a.y, P);            // R = S2 - Y1
    if (fp381_is_zero(pp)) {
        if (fp381_is_zero(r)) xyzz_dbl(a, P);
        else xyzz_inf(a);
        return;
    }
    fp381_mul(t, pp, pp, P);
    fp381_mul(ppp, pp, t, P);           // PPP = P^3
    fp381_mul(q, a.x, t, P);            // Q = X1 PP
    fp381_mul(pp, a.zz, t, P);
    fp381_set(a.zz, pp);                // ZZ3 = ZZ1 PP
    fp381_mul(t, a.zzz, ppp, P);
    fp381_set(a.zzz, t);                // ZZZ3 = ZZZ1 PPP
    fp381_mul(t, r, r, P);
    fp381_sub(t, t, ppp, P);
    fp381_sub(t, t, q, P);
    fp381_sub(a.x, t, q, P);            // X3 = R^2 - PPP - 2 Q
    fp381_sub(t, q, a.x, P);
    fp381_mul(q, r, t, P);
    fp381_mul(t, a.y, ppp, P);
    fp381_sub(a.y, q, t, P);            // Y3 = R (Q - X3) - Y1 PPP
}

// a += b, add-2008-s, with the same exceptional cases
CW_HD void xyzz_add(Xyzz381 &a, const Xyzz381 &b, const Fp381Params &P) {
    if (xyzz_is_inf(b)) return;
    if (xyzz_is_inf(a)) {
        a = b;
        return;
    }
    u32 u1[12], s1[12], pp[12], r[12], ppp[12], q[12], t[12];
    fp381_mul(u1, a.x, b.zz, P);
    fp381_mul(t, b.x, a.zz, P);
    fp381_sub(pp, t, u1, P);            // P = U2 - U1
    fp381_mul(s1, a.y, b.zzz, P);
    fp381_mul(t, b.y, a.zzz, P);
    fp381_sub(r, t, s1, P);             // R = S2 - S1
    if (fp381_is_zero(pp)) {
        if (fp381_is_zero(r)) xyzz_dbl(a, P);
        else xyzz_inf(a);
        return;
    }
    fp381_mul(t, pp, pp, P);
    fp381_mul(ppp, pp, t, P);
    fp381_mul(q, u1, t, P);
    fp381_mul(u1, a.zz, b.zz, P);
    fp381_mul(a.zz, u1, t, P);          // ZZ3 = ZZ1 ZZ2 PP
    fp381_mul(u1, a.zzz, b.zzz, P);
    fp381_mul(a.zzz, u1, ppp, P);       // ZZZ3 = ZZZ1 ZZZ2 PPP
    fp381_mul(t, r, r, P);
    fp381_sub(t, t, ppp, P);
    fp381_sub(t, t, q, P);
    fp381_sub(a.x, t, q, P);
    fp381_sub(t, q, a.x, P);
    fp381_mul(q, r, t, P);
    fp381_mul(t, s1, ppp, P);
    fp381_sub(a.y, q, t, P);            // Y3 = R (Q - X3) - S1 PPP
}

// affine Montgomery coordinates of p, (0, 0) for infinity: one inversion of ZZ ZZZ
CW_HD void xyzz_to_affine(u32 *x, u32 *y, const Xyzz381 &p, const Fp381Params &P) {
    if (xyzz_is_inf(p)) {
        fp381_set_u32(x, 0);
        fp381_set_u32(y, 0);
        return;
    }
    u32 t[12], inv[12], s[12];
    fp381_mul(t, p.zz, p.zzz, P);
    fp381_inv(inv, t, P);               // 1 / (ZZ ZZZ)
    fp381_mul(s, inv, p.zzz, P);        // 1 / ZZ
    fp381_mul(x, p.x, s, P);
    fp381_mul(s, inv, p.zz, P);         // 1 / ZZZ
    fp381_mul(y, p.y, s, P);
}

CW_HD void msm_ld_xyzz(Xyzz381 &p, const Xyzz381 *src) {
    const u32 *s = (const u32 *)src;
    fp381_ld(p.x, s);
    fp381_ld(p.y, s + 12);
    fp381_ld(p.zz, s + 24);
    fp381_ld(p.zzz, s + 36);
}

// canonical affine (x, y), 12 limbs each, to Montgomery images: 0 on the curve or (0, 0), 1 a coordinate not below q,
// 2 not on the curve (the host checks of the ABI)
CW_HD int bls12381_g1_to_mont(u32 *xm, u32 *ym, const u32 *x, const u32 *y, const Fp381Params &P) {
    if (fp381_is_zero(x) && fp381_is_zero(y)) {
        fp381_set_u32(xm, 0);
        fp381_set_u32(ym, 0);
        return 0;
    }
    if (!fp381_lt_q(x, P) || !fp381_lt_q(y, P)) return 1;
    u32 b[12], lhs[12], rhs[12];
    fp381_to_mont(xm, x, P);
    fp381_to_mont(ym, y, P);
    fp381_set_u32(b, BLS12381_B);
    fp381_to_mont(b, b, P);
    fp381_mul(lhs, ym, ym, P);
    fp381_mul(rhs, xm, xm, P);
    fp381_mul(rhs, rhs, xm, P);
    fp381_add(rhs, rhs, b, P);
    return fp381_eq(lhs, rhs) ? 0 : 2;
}

// the items of the first level: sorted (key, point index | sign << 31) over the affine bases [n][24] u32
struct MsmBlsAffineItems {
    const u32 *keys, *vals, *bases;
    CW_HD void add(Xyzz381 &acc, uint64_t i, const Fp381Params &P) const {
        const u32 v = vals[i];
        u32 x[12], y[12];
        const u32 *b = bases + 24 * (size_t)(v & 0x7FFFFFFFu);
        fp381_ld(x, b);
        fp381_ld(y, b + 12);
        if (v >> 31) fp381_neg(y, y, P);
        xyzz_madd(acc, x, y, P);
    }
};
// the items of the later levels: partial sums left by the level before
struct MsmBlsXyzzItems {
    const u32 *keys;
    const Xyzz381 *pts;
    CW_HD void add(Xyzz381 &acc, uint64_t i, const Fp381Params &P) const {
        Xyzz381 p;
        msm_ld_xyzz(p, pts + i);
        xyzz_add(acc, p, P);
    }
};

}  // namespace cw

#if defined(__CUDACC__) && !defined(CW_MSM_NO_BLS_G1_KERNELS)   // (msm_bls12381_g2.cu uses the field functions only)
// ---- kernels (sm_90a) -------------------------------------------------------------------------------------------------
// The digits and the sort are msm.cuh's (they do not depend on the group).  The bucket type is 1.5 times the BN254 G1
// one over a product with 2.25 times the limb products, so the kernels run MSM_BLS_THREADS threads per CTA, which lets
// ptxas use up to 255 registers per thread (DESIGN section 4).
namespace cw {

constexpr u32 MSM_BLS_THREADS = 128;

__constant__ Fp381Params c_fp381;

template <bool AFFINE>
__global__ void __launch_bounds__(MSM_BLS_THREADS) msm_bls_runs_kernel(const u32 *__restrict__ keys, const u32 *__restrict__ vals,
                                                                       const u32 *__restrict__ bases,
                                                                       const Xyzz381 *__restrict__ pts, uint64_t N, u32 c,
                                                                       Xyzz381 *buckets, u32 *okeys, Xyzz381 *opts) {
    const Fp381Params &P = c_fp381;
    const uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= threads) return;
    MsmRunOutT<Xyzz381> o{buckets, okeys, opts};
    if (AFFINE) msm_sum_runs(MsmBlsAffineItems{keys, vals, bases}, N, t, c, o, P);
    else msm_sum_runs(MsmBlsXyzzItems{keys, pts}, N, t, c, o, P);
}

// segment results: thread per (window of the chunk, segment of MSM_SEG buckets)
__global__ void __launch_bounds__(MSM_BLS_THREADS) msm_bls_segments_kernel(const Xyzz381 *__restrict__ buckets, u32 B, u32 n_win,
                                                                           Xyzz381 *__restrict__ segs) {
    const Fp381Params &P = c_fp381;
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n_win * per) return;
    const u32 w = (u32)(t / per), s = (u32)(t % per);
    Xyzz381 r;
    msm_bucket_segment(r, buckets + (size_t)w * B, s * m, m, P);
    segs[t] = r;
}

// window sums: one CTA per window of the chunk adds its `per` segment results
__global__ void __launch_bounds__(MSM_BLS_THREADS) msm_bls_windows_kernel(const Xyzz381 *__restrict__ segs, u32 per,
                                                                          Xyzz381 *__restrict__ wins) {
    __shared__ Xyzz381 sm[MSM_BLS_THREADS];
    const Fp381Params &P = c_fp381;
    Xyzz381 acc, b;
    xyzz_inf(acc);
    for (u32 s = threadIdx.x; s < per; s += MSM_BLS_THREADS) {
        msm_ld_xyzz(b, segs + (size_t)blockIdx.x * per + s);
        xyzz_add(acc, b, P);
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (u32 h = MSM_BLS_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            acc = sm[threadIdx.x];
            xyzz_add(acc, sm[threadIdx.x + h], P);
            sm[threadIdx.x] = acc;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) wins[blockIdx.x] = sm[0];
}

// one thread per instance: Horner's rule over its W window sums, then affine canonical [2][6] u64.  Horner's rule is
// msm_horner's, written as one loop over the c doublings and the addition of each window: with the 12-limb doubling
// inlined, msm_horner's nested loops make the device compiler's front end (cicc 12.9) overflow a default 8 MB stack.
__global__ void __launch_bounds__(MSM_BLS_THREADS) msm_bls_final_kernel(const Xyzz381 *__restrict__ wins, u32 W, u32 c, u32 count,
                                                                        uint4 *__restrict__ out) {
    const Fp381Params &P = c_fp381;
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const Xyzz381 *win = wins + (size_t)i * W;
    Xyzz381 acc, s;
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
    u32 x[12], y[12], v[12];
    xyzz_to_affine(x, y, acc, P);
    uint4 *o = out + 6 * (size_t)i;
    fp381_from_mont(v, x, P);
    for (int k = 0; k < 3; ++k) o[k] = make_uint4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
    fp381_from_mont(v, y, P);
    for (int k = 0; k < 3; ++k) o[3 + k] = make_uint4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}

}  // namespace cw
#endif
