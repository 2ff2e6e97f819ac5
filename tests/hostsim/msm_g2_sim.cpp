// CPU run of the library's G2 multi-scalar multiplication: the Fq2 arithmetic and XYZZ formulas of csrc/msm_g2.cuh, and
// whole MSMs through msm.cuh's signed digits, run summation levels and bucket reduction instantiated for XyzzG2, thread by
// thread in the order the kernels run them, with a stable sort in place of the device radix sort
// (tests/test_g2_msm_cpu.py builds this with a plain C++ compiler).
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

#include "msm_g2.cuh"

using namespace cw;

static FrParams dev_params(const FieldParams &F) {
    FrParams p;
    memset(&p, 0, sizeof(p));
    auto split = [](u32 *dst, const U256 &v) {
        for (int i = 0; i < 4; ++i) {
            dst[2 * i] = (u32)v.v[i];
            dst[2 * i + 1] = (u32)(v.v[i] >> 32);
        }
    };
    split(p.q, F.q);
    split(p.half, F.half);
    split(p.r1, F.r1);
    split(p.r2, F.r2);
    U256 qm2;
    u256_sub(qm2, F.q, u256_from_u64(2));
    split(p.qm2, qm2);
    p.np32 = F.np32;
    p.qbits = F.qbits;
    return p;
}

static const FrParams &params() {
    static const FrParams P = dev_params(make_field(MSM_PRIME));
    return P;
}

// canonical [2][4] u64 <-> Montgomery Fq2
static void fq2_in(Fq2 &r, const uint64_t *a) {
    u32 c[8];
    memcpy(c, a, 32);
    fr_to_mont(r.c0, c, params());
    memcpy(c, a + 4, 32);
    fr_to_mont(r.c1, c, params());
}
static void fq2_out(uint64_t *out, const Fq2 &a) {
    u32 c[8];
    fr_from_mont(c, a.c0, params());
    memcpy(out, c, 32);
    fr_from_mont(c, a.c1, params());
    memcpy(out + 4, c, 32);
}
static bool all_zero(const uint64_t *a, int words) {
    for (int i = 0; i < words; ++i)
        if (a[i]) return false;
    return true;
}

// canonical affine [2][2][4] -> XYZZ with ZZ = z^2, ZZZ = z^3 (z canonical Fq2, nonzero); all zeros -> infinity
static XyzzG2 from_affine(const uint64_t *a, const uint64_t *z) {
    const FrParams &P = params();
    XyzzG2 r;
    if (all_zero(a, 16)) {
        xyzz_inf(r);
        return r;
    }
    Fq2 x, y, zm, zz, zzz;
    fq2_in(x, a);
    fq2_in(y, a + 8);
    fq2_in(zm, z);
    fq2_sqr(zz, zm, P);
    fq2_mul(zzz, zz, zm, P);
    fq2_mul(r.x, x, zz, P);
    fq2_mul(r.y, y, zzz, P);
    r.zz = zz;
    r.zzz = zzz;
    return r;
}

static void to_canonical(uint64_t *out, const XyzzG2 &p) {
    Fq2 x, y;
    xyzz_to_affine(x, y, p, params());
    fq2_out(out, x);
    fq2_out(out + 8, y);
}

// Fq2 ops on canonical [2][4] values: 0 a b, 1 a^2, 2 1 / a, 3 a + b, 4 a - b, 5 -a
extern "C" int msm_g2_sim_fq2(int op, const uint64_t *a, const uint64_t *b, uint64_t *out) {
    const FrParams &P = params();
    Fq2 x, y, r;
    fq2_in(x, a);
    fq2_in(y, b);
    switch (op) {
        case 0: fq2_mul(r, x, y, P); break;
        case 1: fq2_sqr(r, x, P); break;
        case 2: fq2_inv(r, x, P); break;
        case 3: fq2_add(r, x, y, P); break;
        case 4: fq2_sub(r, x, y, P); break;
        case 5: fq2_neg(r, x, P); break;
        default: return -1;
    }
    fq2_out(out, r);
    return 0;
}

// op 0: a + b with b mixed (affine); 1: a + b, both XYZZ; 2: 2 a.  a, b, out: canonical affine [2][2][4]; za, zb: the Z
// of the XYZZ forms, canonical [2][4]
extern "C" int msm_g2_sim_op(int op, const uint64_t *a, const uint64_t *za, const uint64_t *b, const uint64_t *zb,
                             uint64_t *out) {
    const FrParams &P = params();
    XyzzG2 A = from_affine(a, za);
    if (op == 0) {
        Fq2 x, y;
        if (all_zero(b, 16)) {
            fq2_zero(x);
            fq2_zero(y);
        } else {
            fq2_in(x, b);
            fq2_in(y, b + 8);
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

// out[i] = sum_j s_{i,j} Q_j for i < count (scalars [count][n][4], points [n][2][2][4] canonical), through the same steps
// as cw_g2_msm_batch; c = 0 takes msm_window_bits(n)
extern "C" int msm_g2_sim_run(const uint64_t *points, const uint64_t *scalars, uint64_t n, uint32_t count, uint32_t c,
                              uint64_t *out) {
    const FrParams &P = params();
    if (!c) c = msm_window_bits(n);
    const u32 W = msm_windows(c), B = 1u << (c - 1);
    std::vector<u32> bases(32 * n, 0u);
    for (uint64_t j = 0; j < n; ++j) {
        if (all_zero(points + 16 * j, 16)) continue;
        Fq2 x, y;
        fq2_in(x, points + 16 * j);
        fq2_in(y, points + 16 * j + 8);
        memcpy(&bases[32 * j], &x, 64);
        memcpy(&bases[32 * j + 16], &y, 64);
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
    std::vector<XyzzG2> buckets((size_t)count * W * B);
    for (auto &b : buckets) xyzz_inf(b);
    std::vector<u32> lk[2];
    std::vector<XyzzG2> lp[2];
    uint64_t items = N, threads = (N + MSM_RUN - 1) / MSM_RUN;
    lk[0].resize(msm_level_out(items));
    lp[0].resize(msm_level_out(items));
    MsmRunOutT<XyzzG2> o0{buckets.data(), lk[0].data(), lp[0].data()};
    for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmG2AffineItems{sk.data(), sv.data(), bases.data()}, N, t, c, o0, P);
    int lv = 0;
    while (threads > 1) {
        items = msm_level_out(items);
        threads = (items + MSM_RUN - 1) / MSM_RUN;
        lk[lv ^ 1].assign(msm_level_out(items), 0);
        lp[lv ^ 1].resize(msm_level_out(items));
        MsmRunOutT<XyzzG2> o{buckets.data(), lk[lv ^ 1].data(), lp[lv ^ 1].data()};
        for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmG2XyzzItems{lk[lv].data(), lp[lv].data()}, items, t, c, o, P);
        lv ^= 1;
    }
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    std::vector<XyzzG2> wins((size_t)count * W);
    for (u32 w = 0; w < count * W; ++w) {
        xyzz_inf(wins[w]);
        for (u32 s = 0; s < per; ++s) {
            XyzzG2 r;
            msm_bucket_segment(r, &buckets[(size_t)w * B], s * m, m, P);
            xyzz_add(wins[w], r, P);
        }
    }
    for (u32 i = 0; i < count; ++i) {
        XyzzG2 acc;
        msm_horner(acc, &wins[(size_t)i * W], W, c, P);
        to_canonical(out + 16 * i, acc);
    }
    return 0;
}
