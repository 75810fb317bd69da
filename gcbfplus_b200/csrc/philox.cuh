// philox.cuh -- stateless counter-based Gaussian draws (device functions only): Philox4x64-10 (Salmon, Moraes, Dror,
// Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC 2011) and the Box-Muller transform in fp64.
// numpy.random.Philox is the same generator; it increments its counter before each block, so
// Philox(counter=c, key=k).random_raw(4) == philox4x64_10(c + [1, 0, 0, 0], k).
#pragma once
#include <stdint.h>

namespace gcbf {

constexpr uint64_t PHILOX_M0 = 0xD2E7470EE14C6C93ull, PHILOX_M1 = 0xCA5A826395121157ull;
constexpr uint64_t PHILOX_W0 = 0x9E3779B97F4A7C15ull, PHILOX_W1 = 0xBB67AE8584CAA73Bull;

// four 64-bit words of counter c under key k (ten rounds, the key bumped by the Weyl constants between rounds)
__device__ __forceinline__ void philox4x64_10(uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3, uint64_t k0,
                                              uint64_t k1, uint64_t w[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) {
            k0 += PHILOX_W0;
            k1 += PHILOX_W1;
        }
        const uint64_t hi0 = __umul64hi(PHILOX_M0, c0), lo0 = PHILOX_M0 * c0;
        const uint64_t hi1 = __umul64hi(PHILOX_M1, c2), lo1 = PHILOX_M1 * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
    }
    w[0] = c0;
    w[1] = c1;
    w[2] = c2;
    w[3] = c3;
}

// u = ((w >> 11) + 1/2) 2^-53 in (0, 1), exact in fp64
__device__ __forceinline__ double philox_uniform(uint64_t w) { return ((double)(w >> 11) + 0.5) * 0x1p-53; }

// Box-Muller in fp64: z0, z1 from (u0, u1) and z2, z3 from (u2, u3), each rounded to fp32 once
__device__ __forceinline__ void box_muller4(const uint64_t w[4], float z[4]) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const double u0 = philox_uniform(w[2 * p]), u1 = philox_uniform(w[2 * p + 1]);
        const double rad = sqrt(-2.0 * log(u0)), ang = 6.283185307179586 * u1;
        z[2 * p] = (float)(rad * cos(ang));
        z[2 * p + 1] = (float)(rad * sin(ang));
    }
}

// the four standard normals of counter (t, env, agent, block) under key (seed, kind)
__device__ __forceinline__ void normal4(uint64_t seed, uint64_t kind, uint64_t t, uint64_t env, uint64_t agent,
                                        uint64_t block, float z[4]) {
    uint64_t w[4];
    philox4x64_10(t, env, agent, block, seed, kind, w);
    box_muller4(w, z);
}

}  // namespace gcbf
