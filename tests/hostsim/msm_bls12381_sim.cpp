// CPU run of the library's BLS12-381 G1 multi-scalar multiplication: the 381-bit field and XYZZ formulas of
// csrc/msm_bls12381.cuh, and whole MSMs through msm.cuh's signed digits, run summation levels and bucket reduction
// instantiated for Xyzz381, thread by thread in the order the kernels run them, with a stable sort in place of the device
// radix sort (tests/test_bls12381_msm_cpu.py builds this with a plain C++ compiler).
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

#include "msm_bls12381.cuh"

using namespace cw;

static const Fp381Params &params() {
    static const Fp381Params P = fp381_params();
    return P;
}

// canonical [6] u64 <-> Montgomery 12 limbs
static void fp_in(u32 *r, const uint64_t *a) {
    u32 c[12];
    memcpy(c, a, 48);
    fp381_to_mont(r, c, params());
}
static void fp_out(uint64_t *out, const u32 *a) {
    u32 c[12];
    fp381_from_mont(c, a, params());
    memcpy(out, c, 48);
}
static bool all_zero(const uint64_t *a, int words) {
    for (int i = 0; i < words; ++i)
        if (a[i]) return false;
    return true;
}

// field ops on canonical [6] u64 values: 0 a b, 1 1 / a, 2 a + b, 3 a - b, 4 -a, 5 from_mont(to_mont(a)), 6 the raw
// Montgomery product a b 2^-384 of the canonical inputs
extern "C" int bls_sim_fp(int op, const uint64_t *a, const uint64_t *b, uint64_t *out) {
    const Fp381Params &P = params();
    u32 x[12], y[12], r[12];
    if (op == 6) {
        memcpy(x, a, 48);
        memcpy(y, b, 48);
        fp381_mul(r, x, y, P);
        memcpy(out, r, 48);
        return 0;
    }
    fp_in(x, a);
    fp_in(y, b);
    switch (op) {
        case 0: fp381_mul(r, x, y, P); break;
        case 1: fp381_inv(r, x, P); break;
        case 2: fp381_add(r, x, y, P); break;
        case 3: fp381_sub(r, x, y, P); break;
        case 4: fp381_neg(r, x, P); break;
        case 5: fp381_set(r, x); break;
        default: return -1;
    }
    fp_out(out, r);
    return 0;
}

// the host check of the ABI on one canonical point [2][6]: 0 fine, 1 a coordinate >= q, 2 not on the curve
extern "C" int bls_sim_check(const uint64_t *xy) {
    u32 x[12], y[12], xm[12], ym[12];
    memcpy(x, xy, 48);
    memcpy(y, xy + 6, 48);
    return bls12381_g1_to_mont(xm, ym, x, y, params());
}

// canonical affine [2][6] -> XYZZ with ZZ = z^2, ZZZ = z^3 (z canonical, nonzero); (0, 0) -> infinity
static Xyzz381 from_affine(const uint64_t *a, const uint64_t *z) {
    const Fp381Params &P = params();
    Xyzz381 r;
    if (all_zero(a, 12)) {
        xyzz_inf(r);
        return r;
    }
    u32 x[12], y[12], zm[12], zz[12], zzz[12];
    fp_in(x, a);
    fp_in(y, a + 6);
    fp_in(zm, z);
    fp381_mul(zz, zm, zm, P);
    fp381_mul(zzz, zz, zm, P);
    fp381_mul(r.x, x, zz, P);
    fp381_mul(r.y, y, zzz, P);
    fp381_set(r.zz, zz);
    fp381_set(r.zzz, zzz);
    return r;
}

static void to_canonical(uint64_t *out, const Xyzz381 &p) {
    u32 x[12], y[12];
    xyzz_to_affine(x, y, p, params());
    fp_out(out, x);
    fp_out(out + 6, y);
}

// op 0: a + b with b mixed (affine); 1: a + b, both XYZZ; 2: 2 a.  a, b, out: canonical affine [2][6]; za, zb: the Z of
// the XYZZ forms, canonical [6]
extern "C" int bls_sim_op(int op, const uint64_t *a, const uint64_t *za, const uint64_t *b, const uint64_t *zb, uint64_t *out) {
    const Fp381Params &P = params();
    Xyzz381 A = from_affine(a, za);
    if (op == 0) {
        u32 x[12], y[12];
        if (all_zero(b, 12)) {
            fp381_set_u32(x, 0);
            fp381_set_u32(y, 0);
        } else {
            fp_in(x, b);
            fp_in(y, b + 6);
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

// out[i] = sum_j s_{i,j} P_j for i < count (scalars [count][n][4], points [n][2][6] canonical), through the same steps as
// cw_bls12381_g1_msm_batch; c = 0 takes msm_window_bits(n)
extern "C" int bls_sim_run(const uint64_t *points, const uint64_t *scalars, uint64_t n, uint32_t count, uint32_t c,
                           uint64_t *out) {
    const Fp381Params &P = params();
    if (!c) c = msm_window_bits(n);
    const u32 W = msm_windows(c), B = 1u << (c - 1);
    std::vector<u32> bases(24 * n, 0u);
    for (uint64_t j = 0; j < n; ++j)
        if (bls_sim_check(points + 12 * j) == 0 && !all_zero(points + 12 * j, 12)) {
            fp_in(&bases[24 * j], points + 12 * j);
            fp_in(&bases[24 * j + 12], points + 12 * j + 6);
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
    std::vector<Xyzz381> buckets((size_t)count * W * B);
    for (auto &b : buckets) xyzz_inf(b);
    std::vector<u32> lk[2];
    std::vector<Xyzz381> lp[2];
    uint64_t items = N, threads = (N + MSM_RUN - 1) / MSM_RUN;
    lk[0].resize(msm_level_out(items));
    lp[0].resize(msm_level_out(items));
    MsmRunOutT<Xyzz381> o0{buckets.data(), lk[0].data(), lp[0].data()};
    for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmBlsAffineItems{sk.data(), sv.data(), bases.data()}, N, t, c, o0, P);
    int lv = 0;
    while (threads > 1) {
        items = msm_level_out(items);
        threads = (items + MSM_RUN - 1) / MSM_RUN;
        lk[lv ^ 1].assign(msm_level_out(items), 0);
        lp[lv ^ 1].resize(msm_level_out(items));
        MsmRunOutT<Xyzz381> o{buckets.data(), lk[lv ^ 1].data(), lp[lv ^ 1].data()};
        for (uint64_t t = 0; t < threads; ++t) msm_sum_runs(MsmBlsXyzzItems{lk[lv].data(), lp[lv].data()}, items, t, c, o, P);
        lv ^= 1;
    }
    const u32 m = B < MSM_SEG ? B : MSM_SEG, per = B / m;
    std::vector<Xyzz381> wins((size_t)count * W);
    for (u32 w = 0; w < count * W; ++w) {
        xyzz_inf(wins[w]);
        for (u32 s = 0; s < per; ++s) {
            Xyzz381 r;
            msm_bucket_segment(r, &buckets[(size_t)w * B], s * m, m, P);
            xyzz_add(wins[w], r, P);
        }
    }
    for (u32 i = 0; i < count; ++i) {
        Xyzz381 acc;
        msm_horner(acc, &wins[(size_t)i * W], W, c, P);
        to_canonical(out + 12 * i, acc);
    }
    return 0;
}
