// Interpreter builds with the function machine (see tape_calls.h).  Product code: part of libcircom_b200.so.
#define CW_KERNELS_TAPE_ONLY 1
#include "tape_calls.h"

namespace cw {

cudaError_t tape_calls_set_params(const FrParams *table, size_t bytes) { return cudaMemcpyToSymbol(c_fr, table, bytes); }

// every build of this unit has the function machine
template <int PR, bool BP, int BT, bool FU>
static bool launch_k(const TapeBuild &k, const TapeLaunch &a) {
    return launch_tape_k<PR, true, BP, BT, FU>(k, a);
}

bool launch_tape_calls(const TapeBuild &k, const TapeLaunch &a) {
    return with_prime(k.prime, [&](auto pr) {
        constexpr int PR = decltype(pr)::value;
        if constexpr (PR >= 0)
            return launch_k<PR, true, 5, false>(k, a) || launch_k<PR, true, -1, false>(k, a) || launch_k<PR, false, -1, false>(k, a);
        else
            return launch_k<-1, true, -1, false>(k, a);
    });
}

}  // namespace cw
