// Multi-scalar multiplication on G1 of BN254 (y^2 = x^3 + 3 over the base field q, the library's `grumpkin` prime):
// the curve formulas, the signed-digit decomposition, the run summation and the bucket reduction (host and device), and
// the kernels that run them (CUDA builds only).  Tests compile the host part with a plain C++ compiler and run whole MSMs
// on the CPU through the same functions (tests/hostsim/msm_sim.cpp).
//
// Pippenger's bucket method with signed c-bit digits: s = sum_w d_w 2^(c w), |d_w| <= 2^(c-1), W = 256 / c + 1 windows
// (the last one takes the carry out of bit 255).  Per (instance, window) every point with d != 0 goes into bucket |d|,
// negated when d < 0; window sum S_w = sum_j j B_j; result = sum_w 2^(c w) S_w by Horner's rule.
//
//   digits   one key (segment = instance * W + window, bucket |d|) and one value (point index | sign << 31) per point and
//            window, then a radix sort of the keys (CUB) puts each bucket's points next to each other.
//   runs     the sorted items are cut into ranges of MSM_RUN; one thread sums the runs of equal keys in its range.  A run
//            that lies inside the range is a whole bucket and is stored; the (at most two) runs that continue into a
//            neighbouring range leave partial sums in two slots per thread, which the next level sums the same way.
//            Each level divides the items by MSM_RUN / 2, so a bucket of n/2 points costs what n/2 spread points cost.
//   buckets  per window, segments of MSM_SEG buckets: running sums from the top give sum (j - lo + 1) B_j and sum B_j,
//            plus lo * sum B_j; a CTA per window adds the segment results; one thread per instance runs Horner's rule
//            and converts to affine with one inversion.
//
// Field elements are Montgomery images mod q (CW_FR index 2).  Buckets are XYZZ (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2);
// the point at infinity is ZZ = ZZZ = 0, so zeroed memory is a row of empty buckets.  Affine bases are (x, y) with
// (0, 0) for infinity (not on the curve: 0 != 3).
#pragma once
#include <stdint.h>

#include "fr_device.cuh"
#include "ntt.cuh"

namespace cw {

constexpr int MSM_PRIME = 2;      // the base field of BN254 G1 in the prime tables
constexpr u32 MSM_RUN = 32;       // sorted items per thread of a run-summing level
constexpr u32 MSM_SEG = 16;       // buckets per thread of the window reduction
constexpr u32 MSM_NONE = 0xFFFFFFFFu;
constexpr u32 MSM_MIN_C = 2, MSM_MAX_C = 18;

struct alignas(16) Xyzz {
    u32 x[8], y[8], zz[8], zzz[8];
};

CW_HD void xyzz_inf(Xyzz &p) {
    u256_set_u32(p.x, 0); u256_set_u32(p.y, 0); u256_set_u32(p.zz, 0); u256_set_u32(p.zzz, 0);
}
CW_HD bool xyzz_is_inf(const Xyzz &p) { return u256_is_zero(p.zz); }

// dbl-2008-s-1 (a = 0): 2M + 5S + the conversions; infinity stays infinity (ZZ = 0).  G1 has odd order, so y != 0.
CW_HD void xyzz_dbl(Xyzz &p, const FrParams &P) {
    u32 u[8], v[8], w[8], s[8], m[8], t[8];
    fr_add(u, p.y, p.y, P);
    fr_mont_mul(v, u, u, P);
    fr_mont_mul(w, u, v, P);
    fr_mont_mul(s, p.x, v, P);
    fr_mont_mul(t, p.x, p.x, P);
    fr_add(m, t, t, P);
    fr_add(m, m, t, P);                 // M = 3 X^2
    fr_mont_mul(t, m, m, P);
    fr_sub(t, t, s, P);
    fr_sub(p.x, t, s, P);               // X3 = M^2 - 2 S
    fr_sub(t, s, p.x, P);
    fr_mont_mul(s, m, t, P);
    fr_mont_mul(t, w, p.y, P);
    fr_sub(p.y, s, t, P);               // Y3 = M (S - X3) - W Y1
    fr_mont_mul(t, v, p.zz, P);
    u256_set(p.zz, t);
    fr_mont_mul(t, w, p.zzz, P);
    u256_set(p.zzz, t);
}

// acc += (x2, y2) affine, madd-2008-s (8M + 2S).  Equal points double, opposite points give infinity; (0, 0) is infinity.
CW_HD void xyzz_madd(Xyzz &a, const u32 *x2, const u32 *y2, const FrParams &P) {
    if (u256_is_zero(x2) && u256_is_zero(y2)) return;
    if (xyzz_is_inf(a)) {
        u256_set(a.x, x2); u256_set(a.y, y2); u256_set(a.zz, P.r1); u256_set(a.zzz, P.r1);
        return;
    }
    u32 pp[8], r[8], ppp[8], q[8], t[8];
    fr_mont_mul(t, x2, a.zz, P);
    fr_sub(pp, t, a.x, P);              // P = U2 - X1
    fr_mont_mul(t, y2, a.zzz, P);
    fr_sub(r, t, a.y, P);               // R = S2 - Y1
    if (u256_is_zero(pp)) {
        if (u256_is_zero(r)) xyzz_dbl(a, P);
        else xyzz_inf(a);
        return;
    }
    fr_mont_mul(t, pp, pp, P);
    fr_mont_mul(ppp, pp, t, P);         // PPP = P^3
    fr_mont_mul(q, a.x, t, P);          // Q = X1 PP
    fr_mont_mul(pp, a.zz, t, P);
    u256_set(a.zz, pp);                 // ZZ3 = ZZ1 PP
    fr_mont_mul(t, a.zzz, ppp, P);
    u256_set(a.zzz, t);                 // ZZZ3 = ZZZ1 PPP
    fr_mont_mul(t, r, r, P);
    fr_sub(t, t, ppp, P);
    fr_sub(t, t, q, P);
    fr_sub(a.x, t, q, P);               // X3 = R^2 - PPP - 2 Q
    fr_sub(t, q, a.x, P);
    fr_mont_mul(q, r, t, P);
    fr_mont_mul(t, a.y, ppp, P);
    fr_sub(a.y, q, t, P);               // Y3 = R (Q - X3) - Y1 PPP
}

// a += b, add-2008-s (12M + 2S), with the same exceptional cases
CW_HD void xyzz_add(Xyzz &a, const Xyzz &b, const FrParams &P) {
    if (xyzz_is_inf(b)) return;
    if (xyzz_is_inf(a)) {
        a = b;
        return;
    }
    u32 u1[8], s1[8], pp[8], r[8], ppp[8], q[8], t[8];
    fr_mont_mul(u1, a.x, b.zz, P);
    fr_mont_mul(t, b.x, a.zz, P);
    fr_sub(pp, t, u1, P);               // P = U2 - U1
    fr_mont_mul(s1, a.y, b.zzz, P);
    fr_mont_mul(t, b.y, a.zzz, P);
    fr_sub(r, t, s1, P);                // R = S2 - S1
    if (u256_is_zero(pp)) {
        if (u256_is_zero(r)) xyzz_dbl(a, P);
        else xyzz_inf(a);
        return;
    }
    fr_mont_mul(t, pp, pp, P);
    fr_mont_mul(ppp, pp, t, P);
    fr_mont_mul(q, u1, t, P);
    fr_mont_mul(u1, a.zz, b.zz, P);
    fr_mont_mul(a.zz, u1, t, P);        // ZZ3 = ZZ1 ZZ2 PP
    fr_mont_mul(u1, a.zzz, b.zzz, P);
    fr_mont_mul(a.zzz, u1, ppp, P);     // ZZZ3 = ZZZ1 ZZZ2 PPP
    fr_mont_mul(t, r, r, P);
    fr_sub(t, t, ppp, P);
    fr_sub(t, t, q, P);
    fr_sub(a.x, t, q, P);
    fr_sub(t, q, a.x, P);
    fr_mont_mul(q, r, t, P);
    fr_mont_mul(t, s1, ppp, P);
    fr_sub(a.y, q, t, P);               // Y3 = R (Q - X3) - S1 PPP
}

// r = k p for a small k (double-and-add from the top bit); Pt: Xyzz here, XyzzG2 in msm_g2.cuh, Xyzz381 in
// msm_bls12381.cuh (the point functions are found by overloading); Par: the field's parameter record (FrParams, or
// Fp381Params for the 381-bit field)
template <class Pt, class Par>
CW_HD void xyzz_mul_small(Pt &r, const Pt &p, u32 k, const Par &P) {
    xyzz_inf(r);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int i = 31; i >= 0; --i) {
        if (!xyzz_is_inf(r)) xyzz_dbl(r, P);
        if ((k >> i) & 1u) xyzz_add(r, p, P);
    }
}

// affine Montgomery coordinates of p, (0, 0) for infinity: one inversion of ZZ ZZZ
CW_HD void xyzz_to_affine(u32 *x, u32 *y, const Xyzz &p, const FrParams &P) {
    if (xyzz_is_inf(p)) {
        u256_set_u32(x, 0);
        u256_set_u32(y, 0);
        return;
    }
    u32 t[8], inv[8], s[8];
    fr_mont_mul(t, p.zz, p.zzz, P);
    fr_inv_mont(inv, t, P);             // 1 / (ZZ ZZZ)
    fr_mont_mul(s, inv, p.zzz, P);      // 1 / ZZ
    fr_mont_mul(x, p.x, s, P);
    fr_mont_mul(s, inv, p.zz, P);       // 1 / ZZZ
    fr_mont_mul(y, p.y, s, P);
}

// ---- the plan ---------------------------------------------------------------------------------------------------------
CW_HD u32 msm_windows(u32 c) { return 256u / c + 1u; }

// the window width: the c in [MSM_MIN_C, MSM_MAX_C] that minimises W (n + 6 * 2^(c-1)): the mixed additions of the
// points plus the two full additions per bucket of the running sums, weighted 6: the sweep of DESIGN section 7 (2^20 and
// 2^21 points on an H100) found the windows one or two bits narrower than a weight of 3 chose 2-7 % faster)
CW_HD u32 msm_window_bits(uint64_t n) {
    u32 best = MSM_MIN_C;
    uint64_t best_cost = ~0ull;
    for (u32 c = MSM_MIN_C; c <= MSM_MAX_C; ++c) {
        const uint64_t cost = (uint64_t)msm_windows(c) * (n + 6ull * (1ull << (c - 1)));
        if (cost < best_cost) {
            best_cost = cost;
            best = c;
        }
    }
    return best;
}

// the next signed digit of the scalar held in t (shifted down by c per call); carry in and out
CW_HD int msm_next_digit(u32 *t, u32 c, u32 &carry) {
    const u32 raw = (t[0] & ((1u << c) - 1u)) + carry;
    u256_shr(t, t, c);
    if (raw > (1u << (c - 1))) {
        carry = 1;
        return (int)raw - (int)(1u << c);
    }
    carry = 0;
    return (int)raw;
}

CW_HD bool msm_live(u32 key, u32 c) { return key != MSM_NONE && (key & ((1u << c) - 1u)) != 0u; }
// bucket slot of a live key: segment * 2^(c-1) + |d| - 1
CW_HD uint64_t msm_slot(u32 key, u32 c) { return ((uint64_t)(key >> c) << (c - 1)) + (key & ((1u << c) - 1u)) - 1u; }

CW_HD void msm_ld_xyzz(Xyzz &p, const Xyzz *src) {
    const u32 *s = (const u32 *)src;
    ntt_ld8(p.x, s);
    ntt_ld8(p.y, s + 8);
    ntt_ld8(p.zz, s + 16);
    ntt_ld8(p.zzz, s + 24);
}

// the items of the first level: sorted (key, point index | sign << 31) over the affine bases [n][16] u32
struct MsmAffineItems {
    const u32 *keys, *vals, *bases;
    CW_HD void add(Xyzz &acc, uint64_t i, const FrParams &P) const {
        const u32 v = vals[i];
        u32 x[8], y[8];
        const u32 *b = bases + 16 * (size_t)(v & 0x7FFFFFFFu);
        ntt_ld8(x, b);
        ntt_ld8(y, b + 8);
        if (v >> 31) fr_neg(y, y, P);
        xyzz_madd(acc, x, y, P);
    }
};
// the items of the later levels: partial sums left by the level before
struct MsmXyzzItems {
    const u32 *keys;
    const Xyzz *pts;
    CW_HD void add(Xyzz &acc, uint64_t i, const FrParams &P) const {
        Xyzz p;
        msm_ld_xyzz(p, pts + i);
        xyzz_add(acc, p, P);
    }
};

// one run's sum at the end of a thread's range walk: a whole bucket goes to `buckets`, a run that continues past the
// range goes to the thread's slot (first run: slot 0, last run: slot 1).  The run machinery below does not depend on the
// group: Pt is the bucket type (Xyzz for G1, XyzzG2 for G2 in msm_g2.cuh, Xyzz381 for BLS12-381 G1 in msm_bls12381.cuh)
// and Par the parameter record its field functions take.
template <class Pt>
struct MsmRunOutT {
    Pt *buckets;
    u32 *okeys;
    Pt *opts;
};
using MsmRunOut = MsmRunOutT<Xyzz>;
template <class Pt>
CW_HD void msm_emit(const MsmRunOutT<Pt> &o, uint64_t t, u32 c, u32 key, const Pt &acc, bool first, bool last, u32 before,
                    u32 after, u32 *slot_key) {
    if (!msm_live(key, c)) return;
    const bool open = (first && key == before) || (last && key == after);
    if (!open) {
        o.buckets[msm_slot(key, c)] = acc;
    } else if (first) {
        o.opts[2 * t] = acc;
        slot_key[0] = key;
        if (last) {   // the range is one run: slot 1 keeps the key (partials of a key stay adjacent) with nothing in it
            Pt z;
            xyzz_inf(z);
            o.opts[2 * t + 1] = z;
            slot_key[1] = key;
        }
    } else {
        o.opts[2 * t + 1] = acc;
        slot_key[1] = key;
    }
}

// thread t of a level over N sorted items: sums the runs of [t MSM_RUN, (t + 1) MSM_RUN)
template <class Items, class Pt, class Par>
CW_HD void msm_sum_runs(const Items &it, uint64_t N, uint64_t t, u32 c, const MsmRunOutT<Pt> &o, const Par &P) {
    const uint64_t lo = t * MSM_RUN, hi = lo + MSM_RUN < N ? lo + MSM_RUN : N;
    const u32 before = lo > 0 ? it.keys[lo - 1] : MSM_NONE, after = hi < N ? it.keys[hi] : MSM_NONE;
    u32 slot_key[2] = {MSM_NONE, MSM_NONE};
    u32 cur = it.keys[lo];
    bool first = true;
    Pt acc;
    xyzz_inf(acc);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (uint64_t i = lo; i < hi; ++i) {
        const u32 k = it.keys[i];
        if (k != cur) {
            msm_emit(o, t, c, cur, acc, first, false, before, after, slot_key);
            first = false;
            cur = k;
            xyzz_inf(acc);
        }
        if (msm_live(k, c)) it.add(acc, i, P);
    }
    msm_emit(o, t, c, cur, acc, first, true, before, after, slot_key);
    o.okeys[2 * t] = slot_key[0];
    o.okeys[2 * t + 1] = slot_key[1];
}

// slots after a level over N items
CW_HD uint64_t msm_level_out(uint64_t N) { return 2 * ((N + MSM_RUN - 1) / MSM_RUN); }

// buckets [lo, lo + m) of one window (bucket b holds digit b + 1): sum_{b} (b + 1) B_b over the segment
template <class Pt, class Par>
CW_HD void msm_bucket_segment(Pt &out, const Pt *win, u32 lo, u32 m, const Par &P) {
    Pt run, tot, b;
    xyzz_inf(run);
    xyzz_inf(tot);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (u32 j = lo + m; j-- > lo;) {
        msm_ld_xyzz(b, win + j);
        xyzz_add(run, b, P);
        xyzz_add(tot, run, P);          // tot = sum (j - lo + 1) B_j
    }
    xyzz_mul_small(out, run, lo, P);
    xyzz_add(out, tot, P);
}

// sum_w 2^(c w) S_w (Horner's rule from the top window)
template <class Pt, class Par>
CW_HD void msm_horner(Pt &acc, const Pt *win, u32 W, u32 c, const Par &P) {
    msm_ld_xyzz(acc, win + (W - 1));
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (u32 w = W - 1; w-- > 0;) {
        for (u32 k = 0; k < c; ++k) xyzz_dbl(acc, P);
        Pt s;
        msm_ld_xyzz(s, win + w);
        xyzz_add(acc, s, P);
    }
}

}  // namespace cw

#if defined(__CUDACC__)
// ---- kernels (sm_90a) -------------------------------------------------------------------------------------------------
#include "kernels.cuh"

namespace cw {

constexpr u32 MSM_THREADS = 256;

// (the G2 unit, msm_g2.cu, includes this header for the shared functions and defines CW_MSM_NO_G1_KERNELS: the
// non-template kernels must exist in one translation unit only)
#ifndef CW_MSM_NO_G1_KERNELS

// keys and values of `count` instances: item (instance i, window w, point j) at (i W + w) n + j.  grid.y = instances.
__global__ void __launch_bounds__(MSM_THREADS) msm_digits_kernel(const uint4 *__restrict__ scalars, uint64_t stride_elems,
                                                                 u32 n, u32 c, u32 W, u32 count, u32 *__restrict__ keys,
                                                                 u32 *__restrict__ vals) {
    for (u32 i = blockIdx.y; i < count; i += gridDim.y) {
        for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
            u32 t[8];
            ldg256_nc(t, scalars + 2 * (i * stride_elems + j));
            u32 carry = 0;
#pragma unroll 1
            for (u32 w = 0; w < W; ++w) {
                const int d = msm_next_digit(t, c, carry);
                const u32 seg = i * W + w;
                const size_t at = (size_t)seg * n + j;
                keys[at] = (seg << c) | (u32)(d < 0 ? -d : d);
                vals[at] = j | (d < 0 ? 0x80000000u : 0u);
            }
        }
    }
}

template <bool AFFINE>
__global__ void __launch_bounds__(MSM_THREADS) msm_runs_kernel(const u32 *__restrict__ keys, const u32 *__restrict__ vals,
                                                               const u32 *__restrict__ bases, const Xyzz *__restrict__ pts,
                                                               uint64_t N, u32 c, Xyzz *buckets, u32 *okeys, Xyzz *opts) {
    const FrParams &P = c_fr[MSM_PRIME];
    const uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= threads) return;
    MsmRunOut o{buckets, okeys, opts};
    if (AFFINE) msm_sum_runs(MsmAffineItems{keys, vals, bases}, N, t, c, o, P);
    else msm_sum_runs(MsmXyzzItems{keys, pts}, N, t, c, o, P);
}

// segment results: thread per (window of the chunk, segment of MSM_SEG buckets); B = 2^(c-1) buckets per window
__global__ void __launch_bounds__(MSM_THREADS) msm_segments_kernel(const Xyzz *__restrict__ buckets, u32 B, u32 n_win,
                                                                   Xyzz *__restrict__ segs) {
    const FrParams &P = c_fr[MSM_PRIME];
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n_win * per) return;
    const u32 w = (u32)(t / per), s = (u32)(t % per);
    Xyzz r;
    msm_bucket_segment(r, buckets + (size_t)w * B, s * m, m, P);
    segs[t] = r;
}

// window sums: one CTA per window of the chunk adds its `per` segment results
__global__ void __launch_bounds__(MSM_THREADS) msm_windows_kernel(const Xyzz *__restrict__ segs, u32 per, Xyzz *__restrict__ wins) {
    __shared__ Xyzz sm[MSM_THREADS];
    const FrParams &P = c_fr[MSM_PRIME];
    Xyzz acc, b;
    xyzz_inf(acc);
    for (u32 s = threadIdx.x; s < per; s += MSM_THREADS) {
        msm_ld_xyzz(b, segs + (size_t)blockIdx.x * per + s);
        xyzz_add(acc, b, P);
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (u32 h = MSM_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            acc = sm[threadIdx.x];
            xyzz_add(acc, sm[threadIdx.x + h], P);
            sm[threadIdx.x] = acc;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) wins[blockIdx.x] = sm[0];
}

// one thread per instance: Horner's rule over its W window sums, then affine canonical [2][4] u64
__global__ void __launch_bounds__(MSM_THREADS) msm_final_kernel(const Xyzz *__restrict__ wins, u32 W, u32 c, u32 count,
                                                                uint4 *__restrict__ out) {
    const FrParams &P = c_fr[MSM_PRIME];
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Xyzz acc;
    msm_horner(acc, wins + (size_t)i * W, W, c, P);
    u32 x[8], y[8], cx[8], cy[8];
    xyzz_to_affine(x, y, acc, P);
    fr_from_mont(cx, x, P);
    fr_from_mont(cy, y, P);
    stg256(out + 4 * (size_t)i, cx);
    stg256(out + 4 * (size_t)i + 2, cy);
}
#endif  // CW_MSM_NO_G1_KERNELS

}  // namespace cw
#endif
