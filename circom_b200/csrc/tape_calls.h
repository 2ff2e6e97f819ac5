// Which build of the interpreter a run lands on, and its launch.  The builds that contain the function machine
// (tape_exec_kernel<.., HAS_CALLS = true, ..>) live in their own translation unit, tape_calls.cu: ptxas does not survive
// one module with every build of the interpreter.
#pragma once
#include <cuda_runtime.h>

#include <type_traits>

#include "kernels.cuh"

namespace cw {
// this unit's copy of the constant field-parameter table (every .cu has its own c_fr without relocatable device code)
cudaError_t tape_calls_set_params(const FrParams *table, size_t bytes);

// f(std::integral_constant<int, PRIME>) for the kernel build of a prime: bn128 and bls12381 have their own (PRIME = 0 / 1),
// the other primes share the build that takes the index at run time (PRIME = -1)
template <class F>
auto with_prime(int prime_id, F &&f) {
    if (prime_id == 0) return f(std::integral_constant<int, 0>{});
    if (prime_id == 1) return f(std::integral_constant<int, 1>{});
    return f(std::integral_constant<int, -1>{});
}

// a build tape_exec_kernel<PRIME, HAS_CALLS, BP, BT, FUSED>: prime -1 = index from TapeDev::prime, bt -1 = tile size from the
// kernel's argument
struct TapeBuild {
    int prime;
    bool calls, bp;
    int bt;
    bool fused;
};

// The build for a tape on prime `prime_id` with / without function calls, a bit plane and fused work items, in tiles of
// 1 << bt_log2 instances; false: there is none (fused work items on a prime without builds of its own).
//   - calls: the builds with the function machine, never fused (the lowering does not fuse tapes with calls: measured
//     slower, flatten.cpp); warp-per-op tiles with a bit plane - the large-batch layout - get the tile size fixed at compile
//     time, everything else takes it as an argument
//   - fused work items (CW_FLAG_FUSE): the bit-plane build (it also runs tapes without a plane: they contain no plane
//     operands), a warp per op or the tile size as an argument
//   - one operator per work item, per bit-plane mode: one instance per tile / a warp per op (tile sizes fixed at compile
//     time) / tile size as an argument
//   - the other 256-bit primes: one build (bit-plane capable, tile size as an argument), with or without calls
inline bool select_tape_build(int prime_id, bool calls, bool bp, bool fused, u32 bt_log2, TapeBuild &k) {
    const int pr = with_prime(prime_id, [](auto p) { return (int)decltype(p)::value; });
    const int bt = (int)bt_log2;
    if (pr < 0) {
        if (fused) return false;
        k = {-1, calls, true, -1, false};
    } else if (calls) k = {pr, true, bp, bp && bt == 5 ? 5 : -1, false};
    else if (fused) k = {pr, false, true, bt == 5 ? 5 : -1, true};
    else if (bp) k = {pr, false, true, bt == 0 || bt == 5 ? bt : -1, false};
    else k = {pr, false, false, bt == 0 ? 0 : -1, false};
    return true;
}

// one launch of the interpreter over the value store of a batch
struct TapeLaunch {
    TapeDev tp;
    uint4 *slots;
    u32 *plane;
    u32 bt_log2;
    u32 *first_assert;
    int *err;
    u32 batch, tiles, threads;
    cudaStream_t stream;
};

// launches tape_exec_kernel<PR, CALLS, BP, BT, FU> if that is the build k names
// (the fused builds keep their accumulators in dynamic shared memory: kernels.cuh TAPE_ACC_SMEM)
template <int PR, bool CALLS, bool BP, int BT, bool FU>
bool launch_tape_k(const TapeBuild &k, const TapeLaunch &a) {
    if (k.prime != PR || k.calls != CALLS || k.bp != BP || k.bt != BT || k.fused != FU) return false;
    constexpr u32 smem = FU ? TAPE_ACC_SMEM : 0u;
    static_assert(TAPE_ACC_SMEM * CW_TAPE_LB <= 48u * 1024u, "the widest CTA stays within the default dynamic shared memory");
    tape_exec_kernel<PR, CALLS, BP, BT, FU><<<a.tiles, a.threads, smem * a.threads, a.stream>>>(
        a.tp, a.slots, a.plane, a.bt_log2, a.first_assert, a.err, a.batch);
    return true;
}

// the builds with k.calls (tape_calls.cu); false: k names a build the library does not contain
bool launch_tape_calls(const TapeBuild &k, const TapeLaunch &a);
}  // namespace cw
