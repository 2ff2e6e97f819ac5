// Batched radix-2 NTT over the library's 256-bit fields: the pass arithmetic (host and device), the pass plan and the
// host-side root / twiddle tables.  The kernels that run the passes are in kernels.cuh; tests compile this header with a
// plain C++ compiler and run whole transforms on the CPU through the same functions.
//
// Data: `count` vectors of n = 2^log_n canonical elements, [vector][point] x 8 u32 limbs.  Twiddles and scale factors
// are Montgomery images, so MontMul(canonical, image) is the canonical product with no conversion.
//
// Transforms (DIF = Gentleman-Sande, natural in -> bit-reversed out; DIT = Cooley-Tukey, bit-reversed in -> natural out):
//   forward  X_j = sum_i x_i w^(ij)           : DIF forward, then an in-place bit reversal
//   inverse  x_i = 1/n sum_j X_j w^(-ij)      : DIF inverse with 1/n folded into its last pass, then the bit reversal
//   coset    X'_j = sum_i xh_i w2n^i w^(ij) with xh = inverse(X): DIF inverse whose last pass multiplies position p by
//            (1/n) w2n^bitrev(p), then DIT forward - the bit-reversed order between the two is never undone.
// A pass runs `b` consecutive stages on tiles of 2^(b + log_g) points held in shared memory as [limb][point]: 2^log_g
// adjacent columns (stride 2^s_lo) of 2^b rows, so a warp's global accesses cover 2^log_g contiguous elements.
#pragma once
#include <stdint.h>

#include "fr_device.cuh"

namespace cw {

constexpr u32 NTT_TILE_LOG = 11;        // points per CTA tile: 2^11 x 32 B = 64 KB of shared memory
constexpr u32 NTT_THREADS = 256;
constexpr u32 NTT_MAX_PASSES = 8;
enum { NTT_SCALE_NONE = 0, NTT_SCALE_CONST = 1, NTT_SCALE_COSET = 2 };
enum { NTT_MODE_FORWARD = 0, NTT_MODE_INVERSE = 1, NTT_MODE_COSET = 2 };

struct NttPass {
    u32 log_n;    // points per vector: 2^log_n
    u32 s_lo, b;  // the stages of half-distance 2^s for s in [s_lo, s_lo + b)
    u32 log_g;    // columns per tile (adjacent groups of the same rows)
    u32 inverse;  // twiddles w^-j
    u32 scale;    // NTT_SCALE_*: after the butterflies of this pass (DIF passes only)
    u32 lg_lo;    // coset scale factor of index i: hi[i >> lg_lo] * lo[i & (2^lg_lo - 1)]
};

CW_HD u32 ntt_bitrev(u32 i, u32 log_n) {
    u32 r = 0;
    for (u32 k = 0; k < log_n; ++k) r |= ((i >> k) & 1u) << (log_n - 1u - k);
    return r;
}

// global point index of tile-local element e of tile `blk`; e = row << log_g | column
CW_HD u32 ntt_gidx(const NttPass &p, u32 blk, u32 e) {
    const u32 g0 = blk << p.log_g;   // first group of the tile
    const u32 lo_mask = (1u << p.s_lo) - 1u;
    const u32 base = ((g0 >> p.s_lo) << (p.s_lo + p.b)) + (g0 & lo_mask);
    return base + ((e >> p.log_g) << p.s_lo) + (e & ((1u << p.log_g) - 1u));
}

CW_HD void ntt_ld8(u32 *v, const u32 *p) {
#if defined(__CUDA_ARCH__)
    const uint4 lo = __ldg((const uint4 *)p), hi = __ldg((const uint4 *)p + 1);
    v[0] = lo.x; v[1] = lo.y; v[2] = lo.z; v[3] = lo.w;
    v[4] = hi.x; v[5] = hi.y; v[6] = hi.z; v[7] = hi.w;
#else
    for (int i = 0; i < 8; ++i) v[i] = p[i];
#endif
}

// butterfly q (of 2^(b + log_g - 1)) of local stage t on the tile in `sm` ([limb][T]).  tw[j] = w^j (Montgomery), j < n/2;
// w^-j = -w^(n/2 - j) for j > 0, so the inverse transform reads the same table and swaps the add and the subtract.
CW_HD void ntt_butterfly(u32 *sm, u32 T, const NttPass &p, u32 blk, u32 t, u32 q, const u32 *tw, bool dit,
                         const FrParams &P) {
    const u32 pb = p.log_g + t;   // local distance of the pair: 2^pb
    const u32 e0 = ((q >> pb) << (pb + 1)) | (q & ((1u << pb) - 1u)), e1 = e0 | (1u << pb);
    const u32 s = p.s_lo + t;
    u32 j = (ntt_gidx(p, blk, e0) & ((1u << s) - 1u)) << (p.log_n - 1u - s);
    bool swap = false;
    if (p.inverse && j) {
        j = (1u << (p.log_n - 1u)) - j;
        swap = true;
    }
    u32 u[8], v[8], r0[8], r1[8];
#pragma unroll
    for (int l = 0; l < 8; ++l) {
        u[l] = sm[l * T + e0];
        v[l] = sm[l * T + e1];
    }
    if (dit) {   // (u, v) -> (u + w v, u - w v)
        if (j) {
            u32 w[8], m[8];
            ntt_ld8(w, tw + 8 * (size_t)j);
            fr_mont_mul(m, v, w, P);
            u256_set(v, m);
        }
        if (swap) {
            fr_sub(r0, u, v, P);
            fr_add(r1, u, v, P);
        } else {
            fr_add(r0, u, v, P);
            fr_sub(r1, u, v, P);
        }
    } else {     // (u, v) -> (u + v, (u - v) w)
        fr_add(r0, u, v, P);
        u32 d[8];
        if (swap) fr_sub(d, v, u, P);
        else fr_sub(d, u, v, P);
        if (j) {
            u32 w[8];
            ntt_ld8(w, tw + 8 * (size_t)j);
            fr_mont_mul(r1, d, w, P);
        } else u256_set(r1, d);
    }
#pragma unroll
    for (int l = 0; l < 8; ++l) {
        sm[l * T + e0] = r0[l];
        sm[l * T + e1] = r1[l];
    }
}

// the scale factor of a DIF pass applied to the value x at global position i (canonical in, canonical out)
CW_HD void ntt_scale(u32 *x, u32 i, const NttPass &p, const u32 *shi, const u32 *slo, const FrParams &P) {
    u32 c[8], r[8];
    if (p.scale == NTT_SCALE_CONST) {
        ntt_ld8(c, shi);
    } else {
        const u32 k = ntt_bitrev(i, p.log_n);   // DIF output position i holds coefficient bitrev(i)
        u32 h[8], l[8];
        ntt_ld8(h, shi + 8 * (size_t)(k >> p.lg_lo));
        ntt_ld8(l, slo + 8 * (size_t)(k & ((1u << p.lg_lo) - 1u)));
        fr_mont_mul(c, h, l, P);   // Montgomery image of the product
    }
    fr_mont_mul(r, x, c, P);
    u256_set(x, r);
}

// h = a * b - c for canonical a, b, c
CW_HD void qap_join(u32 *h, const u32 *a, const u32 *b, const u32 *c, const FrParams &P) {
    u32 am[8], ab[8];
    fr_to_mont(am, a, P);
    fr_mont_mul(ab, am, b, P);
    fr_sub(h, ab, c, P);
}

// The passes of one transform in execution order.  The stages s < min(log_n, NTT_TILE_LOG) form one pass over contiguous
// tiles; the stages above are split evenly into passes of at most NTT_TILE_LOG - 1 stages, whose tiles take at least two
// adjacent columns (64 contiguous bytes per row; 2^(NTT_TILE_LOG - b) columns where the pass is shorter).
// DIF runs from the top stages down, DIT from the bottom up.  Returns the number of passes.
CW_HD u32 ntt_plan(u32 log_n, bool dit, u32 inverse, u32 last_scale, u32 lg_lo, NttPass *out) {
    const u32 b0 = log_n < NTT_TILE_LOG ? log_n : NTT_TILE_LOG;
    const u32 up = log_n - b0;
    const u32 n_up = (up + NTT_TILE_LOG - 2u) / (NTT_TILE_LOG - 1u);
    NttPass ps[NTT_MAX_PASSES];
    u32 np = 0, s = 0;
    ps[np++] = NttPass{log_n, 0u, b0, 0u, inverse, NTT_SCALE_NONE, lg_lo};
    s = b0;
    for (u32 k = 0; k < n_up; ++k) {
        const u32 b = up / n_up + (k < up % n_up ? 1u : 0u);
        u32 lg = NTT_TILE_LOG - b;
        if (lg > s) lg = s;
        ps[np++] = NttPass{log_n, s, b, lg, inverse, NTT_SCALE_NONE, lg_lo};
        s += b;
    }
    // bottom-up order; DIF reverses it and scales in its last pass (the contiguous one)
    for (u32 k = 0; k < np; ++k) out[k] = ps[dit ? k : np - 1u - k];
    if (!dit) out[np - 1u].scale = last_scale;
    return np;
}

}  // namespace cw

// ---- host side: roots of unity and the tables the passes read --------------------------------------------------------
#include <vector>

#include "u256.h"

namespace cw {

// 2-adicity s of q - 1
inline u32 ntt_two_adicity(const FieldParams &F) {
    U256 qm1;
    u256_sub(qm1, F.q, u256_from_u64(1));
    u32 s = 0;
    while (s < 255 && !((qm1.v[s >> 6] >> (s & 63)) & 1)) ++s;
    return s;
}

// x^e, x and result as Montgomery images
inline U256 ntt_pow_mont(const FieldParams &F, const U256 &xm, const U256 &e) {
    U256 r = F.r1, b = xm;
    for (int i = 0; i < 256; ++i) {
        if ((e.v[i >> 6] >> (i & 63)) & 1) r = F.mont_mul(r, b);
        b = F.mont_mul(b, b);
    }
    return r;
}

// Montgomery image of w_{2^j} = g^(t * 2^(s - j)), g the smallest quadratic non-residue counted up from 2, t = (q-1) / 2^s
inline U256 ntt_root_mont(const FieldParams &F, u32 j) {
    const u32 s = ntt_two_adicity(F);
    U256 qm1, half, t;
    u256_sub(qm1, F.q, u256_from_u64(1));
    for (int i = 0; i < 4; ++i) half.v[i] = (qm1.v[i] >> 1) | (i < 3 ? (qm1.v[i + 1] << 63) : 0);
    U256 g = u256_from_u64(2);
    U256 minus1 = F.subm(u256_from_u64(0), F.r1);
    while (ntt_pow_mont(F, F.to_mont(g), half) != minus1) g.v[0] += 1;
    t = qm1;
    for (u32 k = 0; k < s; ++k)
        for (int i = 0; i < 4; ++i) t.v[i] = (t.v[i] >> 1) | (i < 3 ? (t.v[i + 1] << 63) : 0);
    U256 w = ntt_pow_mont(F, F.to_mont(g), t);   // a primitive 2^s-th root
    for (u32 k = j; k < s; ++k) w = F.mont_mul(w, w);
    return w;
}

// tw[j] = w_n^j, j < n/2; shi[h] = (1/n) w_2n^(h << lg_lo); slo[l] = w_2n^l.  shi[0] is the 1/n of the plain inverse.
inline u32 ntt_lg_lo(u32 log_n) { return (log_n + 1u) / 2u; }
inline void ntt_tables(const FieldParams &F, u32 log_n, std::vector<U256> &tw, std::vector<U256> &shi, std::vector<U256> &slo) {
    const uint64_t n = 1ull << log_n;
    const u32 lg_lo = ntt_lg_lo(log_n);
    const U256 w = ntt_root_mont(F, log_n), w2 = ntt_root_mont(F, log_n + 1);
    tw.resize(n / 2);
    U256 x = F.r1;
    for (uint64_t j = 0; j < n / 2; ++j) {
        tw[j] = x;
        x = F.mont_mul(x, w);
    }
    slo.resize((size_t)1 << lg_lo);
    x = F.r1;
    for (size_t l = 0; l < slo.size(); ++l) {
        slo[l] = x;
        x = F.mont_mul(x, w2);
    }
    // x = w_2n^(2^lg_lo); 1/n = ((q + 1) / 2)^log_n
    U256 inv2;
    {
        U256 qp1;
        u256_add(qp1, F.q, u256_from_u64(1));
        for (int i = 0; i < 4; ++i) inv2.v[i] = (qp1.v[i] >> 1) | (i < 3 ? (qp1.v[i + 1] << 63) : 0);
    }
    U256 inv_n = F.r1;
    const U256 inv2m = F.to_mont(inv2);
    for (u32 k = 0; k < log_n; ++k) inv_n = F.mont_mul(inv_n, inv2m);
    shi.resize((size_t)1 << (log_n - lg_lo));
    U256 y = inv_n;
    for (size_t h = 0; h < shi.size(); ++h) {
        shi[h] = y;
        y = F.mont_mul(y, x);
    }
}

}  // namespace cw
