// CPU run of the library's G1 multi-scalar multiplication: the XYZZ formulas, the signed digits, the run summation
// levels and the bucket reduction of csrc/msm.cuh, executed thread by thread in the order the kernels run them, with a
// stable sort in place of the device radix sort (tests/test_msm_cpu.py builds this with a plain C++ compiler).
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

#include "msm.cuh"

using namespace cw;

static const FrParams &params() {
    static const FrParams P = make_dev_params(make_field(MSM_PRIME));
    return P;
}

// canonical affine (x, y) -> XYZZ with ZZ = z^2, ZZZ = z^3 (z canonical, nonzero); (0, 0) -> infinity
static Xyzz from_affine(const uint64_t *a, const uint64_t *z) {
    const FrParams &P = params();
    Xyzz r;
    u32 x[8], y[8];
    memcpy(x, a, 32);
    memcpy(y, a + 4, 32);
    if (u256_is_zero(x) && u256_is_zero(y)) {
        xyzz_inf(r);
        return r;
    }
    u32 zc[8], zm[8], xm[8], ym[8], zz[8], zzz[8];
    memcpy(zc, z, 32);
    fr_to_mont(zm, zc, P);
    fr_to_mont(xm, x, P);
    fr_to_mont(ym, y, P);
    fr_mont_mul(zz, zm, zm, P);
    fr_mont_mul(zzz, zz, zm, P);
    fr_mont_mul(r.x, xm, zz, P);
    fr_mont_mul(r.y, ym, zzz, P);
    u256_set(r.zz, zz);
    u256_set(r.zzz, zzz);
    return r;
}

static void to_canonical(uint64_t *out, const Xyzz &p) {
    const FrParams &P = params();
    u32 x[8], y[8], cx[8], cy[8];
    xyzz_to_affine(x, y, p, P);
    fr_from_mont(cx, x, P);
    fr_from_mont(cy, y, P);
    memcpy(out, cx, 32);
    memcpy(out + 4, cy, 32);
}

// op 0: a + b with b mixed (affine); 1: a + b, both XYZZ; 2: 2 a.  a, b, out: canonical affine [2][4]; za, zb: the Z of
// the XYZZ forms
extern "C" int msm_sim_op(int op, const uint64_t *a, const uint64_t *za, const uint64_t *b, const uint64_t *zb, uint64_t *out) {
    const FrParams &P = params();
    Xyzz A = from_affine(a, za);
    if (op == 0) {
        u32 x[8], y[8], xm[8], ym[8];
        memcpy(x, b, 32);
        memcpy(y, b + 4, 32);
        if (u256_is_zero(x) && u256_is_zero(y)) {
            u256_set_u32(xm, 0);
            u256_set_u32(ym, 0);
        } else {
            fr_to_mont(xm, x, P);
            fr_to_mont(ym, y, P);
        }
        xyzz_madd(A, xm, ym, P);
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

// the signed digits of one 256-bit scalar in windows of c bits; returns W
extern "C" uint32_t msm_sim_digits(const uint64_t *s, uint32_t c, int32_t *out) {
    u32 t[8], carry = 0;
    memcpy(t, s, 32);
    const u32 W = msm_windows(c);
    for (u32 w = 0; w < W; ++w) out[w] = msm_next_digit(t, c, carry);
    return carry;   // 0: the digits are complete
}

extern "C" uint32_t msm_sim_window_bits(uint64_t n) { return msm_window_bits(n); }

// out[i] = sum_j s_{i,j} P_j for i < count (scalars [count][n][4], points [n][2][4] canonical), through the same steps as
// cw_g1_msm_batch; c = 0 takes msm_window_bits(n)
extern "C" int msm_sim_run(const uint64_t *points, const uint64_t *scalars, uint64_t n, uint32_t count, uint32_t c,
                           uint64_t *out) {
    const FrParams &P = params();
    if (!c) c = msm_window_bits(n);
    const u32 W = msm_windows(c), B = 1u << (c - 1);
    std::vector<u32> bases(16 * n);
    for (uint64_t j = 0; j < n; ++j) {
        u32 x[8], y[8];
        memcpy(x, points + 8 * j, 32);
        memcpy(y, points + 8 * j + 4, 32);
        if (!(u256_is_zero(x) && u256_is_zero(y))) {
            fr_to_mont(&bases[16 * j], x, P);
            fr_to_mont(&bases[16 * j + 8], y, P);
        } else {
            std::fill(&bases[16 * j], &bases[16 * j + 16], 0u);
        }
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
    std::vector<Xyzz> buckets((size_t)count * W * B);
    for (auto &b : buckets) xyzz_inf(b);
    std::vector<u32> lk[2];
    std::vector<Xyzz> lp[2];
    uint64_t items = N, threads = (N + MSM_RUN - 1) / MSM_RUN;
    lk[0].resize(msm_level_out(items));
    lp[0].resize(msm_level_out(items));
    MsmRunOut o0{buckets.data(), lk[0].data(), lp[0].data()};
    for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmAffineItems{sk.data(), sv.data(), bases.data()}, N, t, c, o0, P);
    int lv = 0;
    while (threads > 1) {
        items = msm_level_out(items);
        threads = (items + MSM_RUN - 1) / MSM_RUN;
        lk[lv ^ 1].assign(msm_level_out(items), 0);
        lp[lv ^ 1].resize(msm_level_out(items));
        MsmRunOut o{buckets.data(), lk[lv ^ 1].data(), lp[lv ^ 1].data()};
        for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmXyzzItems{lk[lv].data(), lp[lv].data()}, items, t, c, o, P);
        lv ^= 1;
    }
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    std::vector<Xyzz> wins((size_t)count * W);
    for (u32 w = 0; w < count * W; ++w) {
        xyzz_inf(wins[w]);
        for (u32 s = 0; s < per; ++s) {
            Xyzz r;
            msm_bucket_segment(r, &buckets[(size_t)w * B], s * m, m, P);
            xyzz_add(wins[w], r, P);
        }
    }
    for (u32 i = 0; i < count; ++i) {
        Xyzz acc;
        msm_horner(acc, &wins[(size_t)i * W], W, c, P);
        to_canonical(out + 8 * i, acc);
    }
    return 0;
}
