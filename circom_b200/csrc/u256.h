// Host-side 256-bit helpers and per-prime constants (computed, not tabulated).
// Used by the lowering (Montgomery images of constants) and the file-format code.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>

namespace cw {

struct U256 {
    uint64_t v[4];
    bool operator==(const U256 &o) const { return !memcmp(v, o.v, 32); }
    bool operator!=(const U256 &o) const { return !(*this == o); }
    bool operator<(const U256 &o) const {
        for (int i = 3; i >= 0; --i) {
            if (v[i] != o.v[i]) return v[i] < o.v[i];
        }
        return false;
    }
    bool is_zero() const { return (v[0] | v[1] | v[2] | v[3]) == 0; }
};

inline U256 u256_from_u64(uint64_t x) { return U256{{x, 0, 0, 0}}; }

inline uint64_t u256_add(U256 &r, const U256 &a, const U256 &b) {
    unsigned __int128 c = 0;
    for (int i = 0; i < 4; ++i) {
        c += (unsigned __int128)a.v[i] + b.v[i];
        r.v[i] = (uint64_t)c;
        c >>= 64;
    }
    return (uint64_t)c;
}
inline uint64_t u256_sub(U256 &r, const U256 &a, const U256 &b) {
    unsigned __int128 br = 0;
    for (int i = 0; i < 4; ++i) {
        unsigned __int128 t = (unsigned __int128)a.v[i] - b.v[i] - br;
        r.v[i] = (uint64_t)t;
        br = (t >> 64) & 1;
    }
    return (uint64_t)br;
}

constexpr int CW_N_PRIMES = 8;  // bn128, bls12381, grumpkin, pallas, vesta, secq256r1, bls12377, goldilocks
// id of the prime with modulus q, or -1
int prime_id_of(const struct U256 &q);

// Field constants for one prime.  q from program_structure/src/utils/constants.rs:3-6;
// derived values as the reference compiler derives them (c_code_generator.rs:1086-1099).
struct FieldParams {
    int prime_id;
    U256 q;
    U256 half;     // q >> 1
    U256 r1;       // 2^256 mod q  (Montgomery image of 1)
    U256 r2;       // 2^512 mod q
    uint64_t np64; // -q^-1 mod 2^64
    uint32_t np32; // -q^-1 mod 2^32
    uint32_t qbits;

    U256 addm(const U256 &a, const U256 &b) const {
        U256 r;
        uint64_t c = u256_add(r, a, b);
        if (c || !(r < q)) u256_sub(r, r, q);
        return r;
    }
    U256 subm(const U256 &a, const U256 &b) const {
        U256 r;
        if (u256_sub(r, a, b)) u256_add(r, r, q);
        return r;
    }
    // CIOS Montgomery product a*b*2^-256 mod q (same algorithm as generic/fr.cpp:110-164)
    U256 mont_mul(const U256 &a, const U256 &b) const {
        uint64_t t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 4; ++i) {
            unsigned __int128 c = 0;
            for (int j = 0; j < 4; ++j) {
                c += (unsigned __int128)a.v[j] * b.v[i] + t[j];
                t[j] = (uint64_t)c;
                c >>= 64;
            }
            c += t[4];
            t[4] = (uint64_t)c;
            t[5] = (uint64_t)(c >> 64);
            uint64_t m = t[0] * np64;
            c = (unsigned __int128)m * q.v[0] + t[0];
            c >>= 64;
            for (int j = 1; j < 4; ++j) {
                c += (unsigned __int128)m * q.v[j] + t[j];
                t[j - 1] = (uint64_t)c;
                c >>= 64;
            }
            c += t[4];
            t[3] = (uint64_t)c;
            t[4] = t[5] + (uint64_t)(c >> 64);
        }
        U256 r{{t[0], t[1], t[2], t[3]}};
        if (t[4] || !(r < q)) u256_sub(r, r, q);
        return r;
    }
    U256 to_mont(const U256 &a) const { return mont_mul(a, r2); }
    U256 from_mont(const U256 &a) const { return mont_mul(a, u256_from_u64(1)); }
    U256 mulm(const U256 &a, const U256 &b) const { return mont_mul(to_mont(a), b); }
    // floor(2^(qbits+64) / q) - 2^64: the Barrett constant of fr_mul_small (fr_device.cuh).  The quotient lies in
    // (2^64, 2^65) for any q strictly between two powers of two, so the 64 bits kept here determine it.
    uint64_t barrett_mu() const {
        U256 rem = u256_from_u64(1);
        uint64_t quo = 0;
        for (uint32_t i = 0; i < qbits + 64; ++i) {   // long division of 2^(qbits+64), one bit per step
            const uint64_t carry = u256_add(rem, rem, rem);
            quo <<= 1;
            if (carry || !(rem < q)) {
                u256_sub(rem, rem, q);
                quo |= 1;
            }
        }
        return quo;
    }
};

inline FieldParams make_field(int prime_id) {
    FieldParams f;
    f.prime_id = prime_id;
    // program_structure/src/utils/constants.rs:3-13.  goldilocks (2^64 - 2^32 + 1, c_elements/goldilocks/fr.hpp:11) runs in
    // the same 32-byte elements with six zero limbs: R = 2^256 Montgomery arithmetic holds for any odd modulus
    static const uint64_t Q[CW_N_PRIMES][4] = {
        {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},  // bn128
        {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL},  // bls12381
        {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},  // grumpkin
        {0x992d30ed00000001ULL, 0x224698fc094cf91bULL, 0x0000000000000000ULL, 0x4000000000000000ULL},  // pallas
        {0x8c46eb2100000001ULL, 0x224698fc0994a8ddULL, 0x0000000000000000ULL, 0x4000000000000000ULL},  // vesta
        {0xffffffffffffffffULL, 0x00000000ffffffffULL, 0x0000000000000000ULL, 0xffffffff00000001ULL},  // secq256r1
        {0x0a11800000000001ULL, 0x59aa76fed0000001ULL, 0x60b44d1e5c37b001ULL, 0x12ab655e9a2ca556ULL},  // bls12377
        {0xffffffff00000001ULL, 0x0000000000000000ULL, 0x0000000000000000ULL, 0x0000000000000000ULL},  // goldilocks
    };
    memcpy(f.q.v, Q[prime_id >= 0 && prime_id < CW_N_PRIMES ? prime_id : 0], 32);
    for (int i = 0; i < 4; ++i) f.half.v[i] = (f.q.v[i] >> 1) | (i < 3 ? (f.q.v[i + 1] << 63) : 0);
    // Newton iteration for q^-1 mod 2^64
    uint64_t inv = 1;
    for (int i = 0; i < 6; ++i) inv *= 2 - f.q.v[0] * inv;
    f.np64 = (uint64_t)(0 - inv);
    f.np32 = (uint32_t)f.np64;
    int bits = 0;
    for (int i = 255; i >= 0; --i) {
        if ((f.q.v[i / 64] >> (i % 64)) & 1) { bits = i + 1; break; }
    }
    f.qbits = bits;
    // 2^k mod q by repeated doubling
    U256 x = u256_from_u64(1);
    for (int i = 0; i < 512; ++i) {
        x = f.addm(x, x);
        if (i == 255) f.r1 = x;
    }
    f.r2 = x;
    return f;
}

inline int prime_id_of(const U256 &q) {
    for (int i = 0; i < CW_N_PRIMES; ++i)
        if (make_field(i).q == q) return i;
    return -1;
}

}  // namespace cw
