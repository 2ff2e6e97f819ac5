// CPU run of the library's BLS12-381 G2 multi-scalar multiplication: the Fq2 arithmetic over the 381-bit field and the
// XYZZ formulas of csrc/msm_bls12381_g2.cuh, and whole MSMs through msm.cuh's signed digits, run summation levels and
// bucket reduction instantiated for XyzzG2_381, thread by thread in the order the kernels run them, with a stable sort in
// place of the device radix sort (tests/test_bls12381_g2_msm_cpu.py builds this with a plain C++ compiler).
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

#include "msm_bls12381_g2.cuh"

using namespace cw;

static const Fp381Params &params() {
    static const Fp381Params P = fp381_params();
    return P;
}

// canonical [2][6] u64 (c0, c1) <-> Montgomery Fq2
static void f2_in(Fq2_381 &r, const uint64_t *a) {
    u32 c[12];
    memcpy(c, a, 48);
    fp381_to_mont(r.c0, c, params());
    memcpy(c, a + 6, 48);
    fp381_to_mont(r.c1, c, params());
}
static void f2_out(uint64_t *out, const Fq2_381 &a) {
    u32 c[12];
    fp381_from_mont(c, a.c0, params());
    memcpy(out, c, 48);
    fp381_from_mont(c, a.c1, params());
    memcpy(out + 6, c, 48);
}
static bool all_zero(const uint64_t *a, int words) {
    for (int i = 0; i < words; ++i)
        if (a[i]) return false;
    return true;
}

// Fq2 ops on canonical [2][6] u64 values: 0 a b, 1 1 / a, 2 a + b, 3 a - b, 4 -a, 5 a^2, 6 from_mont(to_mont(a)),
// 7 is_zero(a) (out[0] = 0 / 1)
extern "C" int bls_g2_sim_fq2(int op, const uint64_t *a, const uint64_t *b, uint64_t *out) {
    const Fp381Params &P = params();
    Fq2_381 x, y, r;
    f2_in(x, a);
    f2_in(y, b);
    switch (op) {
        case 0: fq2_mul(r, x, y, P); break;
        case 1: fq2_inv(r, x, P); break;
        case 2: fq2_add(r, x, y, P); break;
        case 3: fq2_sub(r, x, y, P); break;
        case 4: fq2_neg(r, x, P); break;
        case 5: fq2_sqr(r, x, P); break;
        case 6: fq2_set(r, x); break;
        case 7:
            memset(out, 0, 96);
            out[0] = fq2_is_zero(x);
            return 0;
        default: return -1;
    }
    f2_out(out, r);
    return 0;
}

// the host check of the ABI on one canonical point [2][2][6]: 0 fine, 1 a coefficient >= q (*coef: which), 2 not on E'
extern "C" int bls_g2_sim_check(const uint64_t *xy, int *coef) {
    u32 canon[48], mont[48];
    memcpy(canon, xy, 192);
    *coef = -1;
    return bls12381_g2_to_mont(mont, canon, coef, params());
}

// canonical affine [2][2][6] -> XYZZ with ZZ = z^2, ZZZ = z^3 (z canonical [2][6], nonzero); all zeros -> infinity
static XyzzG2_381 from_affine(const uint64_t *a, const uint64_t *z) {
    const Fp381Params &P = params();
    XyzzG2_381 r;
    if (all_zero(a, 24)) {
        xyzz_inf(r);
        return r;
    }
    Fq2_381 x, y, zm, zz, zzz;
    f2_in(x, a);
    f2_in(y, a + 12);
    f2_in(zm, z);
    fq2_sqr(zz, zm, P);
    fq2_mul(zzz, zz, zm, P);
    fq2_mul(r.x, x, zz, P);
    fq2_mul(r.y, y, zzz, P);
    fq2_set(r.zz, zz);
    fq2_set(r.zzz, zzz);
    return r;
}

static void to_canonical(uint64_t *out, const XyzzG2_381 &p) {
    Fq2_381 x, y;
    xyzz_to_affine(x, y, p, params());
    f2_out(out, x);
    f2_out(out + 12, y);
}

// op 0: a + b with b mixed (affine); 1: a + b, both XYZZ; 2: 2 a.  a, b, out: canonical affine [2][2][6]; za, zb: the Z
// of the XYZZ forms, canonical [2][6]
extern "C" int bls_g2_sim_op(int op, const uint64_t *a, const uint64_t *za, const uint64_t *b, const uint64_t *zb,
                             uint64_t *out) {
    const Fp381Params &P = params();
    XyzzG2_381 A = from_affine(a, za);
    if (op == 0) {
        Fq2_381 x, y;
        if (all_zero(b, 24)) {
            fq2_zero(x);
            fq2_zero(y);
        } else {
            f2_in(x, b);
            f2_in(y, b + 12);
        }
        xyzz_madd(A, x, y, P);
    } else if (op == 1) {
        xyzz_add(A, from_affine(b, zb), P);
    } else if (op == 2) {
        xyzz_dbl(A, P);
    } else {
        return -1;
    }
    to_canonical(out, A);
    return 0;
}

// out[i] = sum_j s_{i,j} Q_j for i < count (scalars [count][n][4], points [n][2][2][6] canonical), through the same steps
// as cw_bls12381_g2_msm_batch; c = 0 takes msm_window_bits(n)
extern "C" int bls_g2_sim_run(const uint64_t *points, const uint64_t *scalars, uint64_t n, uint32_t count, uint32_t c,
                              uint64_t *out) {
    const Fp381Params &P = params();
    if (!c) c = msm_window_bits(n);
    const u32 W = msm_windows(c), B = 1u << (c - 1);
    std::vector<u32> bases(48 * n, 0u);
    for (uint64_t j = 0; j < n; ++j) {
        int coef;
        if (bls_g2_sim_check(points + 24 * j, &coef) != 0) return -1;
        u32 canon[48];
        memcpy(canon, points + 24 * j, 192);
        bls12381_g2_to_mont(&bases[48 * j], canon, &coef, P);
    }
    const uint64_t N = (uint64_t)count * W * n;
    std::vector<u32> keys(N), vals(N);
    for (u32 i = 0; i < count; ++i)
        for (uint64_t j = 0; j < n; ++j) {
            u32 t[8], carry = 0;
            memcpy(t, scalars + 4 * (i * n + j), 32);
            for (u32 w = 0; w < W; ++w) {
                const int d = msm_next_digit(t, c, carry);
                const u32 seg = i * W + w;
                keys[(size_t)seg * n + j] = (seg << c) | (u32)(d < 0 ? -d : d);
                vals[(size_t)seg * n + j] = (u32)j | (d < 0 ? 0x80000000u : 0u);
            }
        }
    std::vector<size_t> ord(N);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return keys[a] < keys[b]; });
    std::vector<u32> sk(N), sv(N);
    for (size_t k = 0; k < N; ++k) {
        sk[k] = keys[ord[k]];
        sv[k] = vals[ord[k]];
    }
    std::vector<XyzzG2_381> buckets((size_t)count * W * B);
    for (auto &b : buckets) xyzz_inf(b);
    std::vector<u32> lk[2];
    std::vector<XyzzG2_381> lp[2];
    uint64_t items = N, threads = (N + MSM_RUN - 1) / MSM_RUN;
    lk[0].resize(msm_level_out(items));
    lp[0].resize(msm_level_out(items));
    MsmRunOutT<XyzzG2_381> o0{buckets.data(), lk[0].data(), lp[0].data()};
    for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmBlsG2AffineItems{sk.data(), sv.data(), bases.data()}, N, t, c, o0, P);
    int lv = 0;
    while (threads > 1) {
        items = msm_level_out(items);
        threads = (items + MSM_RUN - 1) / MSM_RUN;
        lk[lv ^ 1].assign(msm_level_out(items), 0);
        lp[lv ^ 1].resize(msm_level_out(items));
        MsmRunOutT<XyzzG2_381> o{buckets.data(), lk[lv ^ 1].data(), lp[lv ^ 1].data()};
        for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmBlsG2XyzzItems{lk[lv].data(), lp[lv].data()}, items, t, c, o, P);
        lv ^= 1;
    }
    // the segment and window sums, then Horner's rule as the final kernel's flat loop runs it
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    std::vector<XyzzG2_381> wins((size_t)count * W);
    for (u32 w = 0; w < count * W; ++w) {
        xyzz_inf(wins[w]);
        for (u32 s = 0; s < per; ++s) {
            XyzzG2_381 r;
            msm_bucket_segment(r, &buckets[(size_t)w * B], s * m, m, P);
            xyzz_add(wins[w], r, P);
        }
    }
    for (u32 i = 0; i < count; ++i) {
        const XyzzG2_381 *win = &wins[(size_t)i * W];
        XyzzG2_381 acc = win[W - 1];
        u32 w = W - 1, k = 0;
        while (w > 0) {
            if (k < c) {
                xyzz_dbl(acc, P);
                ++k;
            } else {
                xyzz_add(acc, win[--w], P);
                k = 0;
            }
        }
        to_canonical(out + 24 * i, acc);
    }
    return 0;
}
