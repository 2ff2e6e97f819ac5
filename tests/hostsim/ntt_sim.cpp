// CPU run of the library's batched NTT: the pass plan, tiles, butterflies and scale factors of csrc/ntt.cuh executed
// tile by tile in the order the kernels run them (tests/test_qap_cpu.py builds this with a plain C++ compiler).
#include <cstring>
#include <vector>

#include "ntt.cuh"

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

static void run_passes(const NttPass *ps, u32 np, bool dit, u32 *vec, const u32 *tw, const u32 *shi, const u32 *slo,
                       const FrParams &P) {
    for (u32 k = 0; k < np; ++k) {
        const NttPass &p = ps[k];
        const u32 T = 1u << (p.b + p.log_g), tiles = 1u << (p.log_n - p.b - p.log_g);
        std::vector<u32> sm(8 * (size_t)T);
        for (u32 blk = 0; blk < tiles; ++blk) {
            for (u32 e = 0; e < T; ++e)
                for (int l = 0; l < 8; ++l) sm[l * (size_t)T + e] = vec[8 * (size_t)ntt_gidx(p, blk, e) + l];
            for (u32 tt = 0; tt < p.b; ++tt) {
                const u32 t = dit ? tt : p.b - 1u - tt;
                for (u32 q = 0; q < T / 2u; ++q) ntt_butterfly(sm.data(), T, p, blk, t, q, tw, dit, P);
            }
            for (u32 e = 0; e < T; ++e) {
                const u32 i = ntt_gidx(p, blk, e);
                u32 r[8];
                for (int l = 0; l < 8; ++l) r[l] = sm[l * (size_t)T + e];
                if (p.scale != NTT_SCALE_NONE) ntt_scale(r, i, p, shi, slo, P);
                for (int l = 0; l < 8; ++l) vec[8 * (size_t)i + l] = r[l];
            }
        }
    }
}

extern "C" int ntt_sim(int prime_id, uint32_t log_n, uint32_t count, uint64_t *data, int mode) {
    const FieldParams F = make_field(prime_id);
    if (log_n < 1 || log_n + 1 > ntt_two_adicity(F)) return -1;
    const FrParams P = dev_params(F);
    std::vector<U256> tw, shi, slo;
    ntt_tables(F, log_n, tw, shi, slo);
    const u32 lg_lo = ntt_lg_lo(log_n);
    NttPass dif[NTT_MAX_PASSES], dit[NTT_MAX_PASSES];
    const u32 scale = mode == NTT_MODE_FORWARD ? NTT_SCALE_NONE : mode == NTT_MODE_INVERSE ? NTT_SCALE_CONST : NTT_SCALE_COSET;
    const u32 nd = ntt_plan(log_n, false, mode != NTT_MODE_FORWARD, scale, lg_lo, dif);
    const u32 nt = ntt_plan(log_n, true, 0u, NTT_SCALE_NONE, lg_lo, dit);
    const u32 n = 1u << log_n;
    for (u32 v = 0; v < count; ++v) {
        u32 *vec = (u32 *)(data + 4 * (size_t)v * n);
        run_passes(dif, nd, false, vec, (const u32 *)tw.data(), (const u32 *)shi.data(), (const u32 *)slo.data(), P);
        if (mode == NTT_MODE_COSET) {
            run_passes(dit, nt, true, vec, (const u32 *)tw.data(), (const u32 *)shi.data(), (const u32 *)slo.data(), P);
        } else {
            for (u32 i = 0; i < n; ++i) {
                const u32 r = ntt_bitrev(i, log_n);
                if (i < r)
                    for (int l = 0; l < 8; ++l) std::swap(vec[8 * (size_t)i + l], vec[8 * (size_t)r + l]);
            }
        }
    }
    return 0;
}

// the pass plan, for the tests: 7 words per pass {log_n, s_lo, b, log_g, inverse, scale, lg_lo}
extern "C" uint32_t ntt_sim_plan(uint32_t log_n, int dit, uint32_t *out) {
    NttPass ps[NTT_MAX_PASSES];
    const u32 np = ntt_plan(log_n, dit != 0, 0u, NTT_SCALE_NONE, ntt_lg_lo(log_n), ps);
    memcpy(out, ps, np * sizeof(NttPass));
    return np;
}
