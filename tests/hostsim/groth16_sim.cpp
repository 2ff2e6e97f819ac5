// CPU run of the library's Groth16 proof assembly (csrc/groth16.cuh): the same functions the kernel calls per (proof,
// group), compiled with a plain C++ compiler (tests/test_groth16_cpu.py builds this).
#include <cstring>

#include "groth16.cuh"

using namespace cw;

static const FrParams &params() {
    static const FrParams P = make_dev_params(make_field(MSM_PRIME));
    return P;
}

// consts: canonical [alpha1 (2), beta1 (2), delta1 (2), beta2 (4), delta2 (4)] x 4 u64; ma, mb1, mc, mh: [2][4], mb2:
// [4][4], rs: [2][4] canonical.  proof: [32] u64 as cw_groth16_prove_* writes it.
extern "C" int g16_sim_assemble(const uint64_t *consts, const uint64_t *ma, const uint64_t *mb1, const uint64_t *mb2,
                                const uint64_t *mc, const uint64_t *mh, const uint64_t *rs, uint64_t *proof) {
    const FrParams &P = params();
    Groth16Consts K;
    u32 *dst[14] = {K.alpha1, K.alpha1 + 8, K.beta1, K.beta1 + 8, K.delta1, K.delta1 + 8,
                    K.beta2, K.beta2 + 8, K.beta2 + 16, K.beta2 + 24, K.delta2, K.delta2 + 8, K.delta2 + 16, K.delta2 + 24};
    for (int k = 0; k < 14; ++k) {
        u32 c[8];
        memcpy(c, consts + 4 * k, 32);
        fr_to_mont(dst[k], c, P);   // (zero stays zero: infinity)
    }
    u32 a[16], b1[16], b2[32], c[16], h[16], r[16], out[64];
    memcpy(a, ma, 64);
    memcpy(b1, mb1, 64);
    memcpy(b2, mb2, 128);
    memcpy(c, mc, 64);
    memcpy(h, mh, 64);
    memcpy(r, rs, 64);
    groth16_g1(out, out + 48, K, a, b1, c, h, r, r + 8, P);
    groth16_g2(out + 16, K, b2, r + 8, P);
    memcpy(proof, out, 256);
    return 0;
}
