// xoshiro.hpp -- the particle jitter generator, shared by the host seeding (hybrid_fluid.cu) and the source emission kernel (flow_kernels.cu).
// rand 0.8.5 `SmallRng` (xoshiro256++ seeded from a u64 through SplitMix64) drawing f32 = (next_u32 >> 8) * 2^-24 with next_u32 = high half
// of next_u64 -- third-party crates that are not vendored in the reference checkout (Cargo.lock: rand 0.8.5, rand_core 0.6.4, cgmath
// 0.18.0); restated from their published algorithms.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define BLUB_HOST_DEVICE __host__ __device__ __forceinline__
#else
#define BLUB_HOST_DEVICE inline
#endif

namespace blub {

struct Xoshiro256pp {
    uint64_t s[4];
    static BLUB_HOST_DEVICE uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    explicit BLUB_HOST_DEVICE Xoshiro256pp(uint64_t state) {
        for (int i = 0; i < 4; ++i) {
            state += 0x9e3779b97f4a7c15ull;
            uint64_t z = state;
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
            s[i] = z ^ (z >> 31);
        }
    }
    BLUB_HOST_DEVICE uint64_t next_u64() {
        const uint64_t result = rotl(s[0] + s[3], 23) + s[0];
        const uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return result;
    }
    // exact: a 24-bit integer times a power of two
    BLUB_HOST_DEVICE float next_f32() { return (float)((uint32_t)(next_u64() >> 32) >> 8) * (1.0f / 16777216.0f); }
};

} // namespace blub
