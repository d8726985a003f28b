// sph_hash.h — the counter-based hash that drives diffuse-particle emission (DESIGN.md section 16).  Plain C++ with integer
// operations only, so the host, the kernels and a float-free restatement (oracle/ref64_diffuse.py) compute the same values.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define SPH_HD __host__ __device__ __forceinline__
#else
#define SPH_HD inline
#endif

// lowbias32 (C. Wellons, "Prospecting for hash functions", 2018): an invertible 32-bit mix
SPH_HD uint32_t sph_mix32(uint32_t x) {
    x ^= x >> 16;
    x *= 0x7feb352du;
    x ^= x >> 15;
    x *= 0x846ca68bu;
    x ^= x >> 16;
    return x;
}

// One word per (seed, update counter, fluid slot, particle id, k, stream); each input is folded in through the mix.  Streams:
// 0 the emission count's rounding u (k = 0), 1 X_r, 2 X_theta and 3 X_h of the k-th particle emitted.
SPH_HD uint32_t sph_diffuse_hash(uint32_t seed, uint32_t counter, uint32_t slot, uint32_t id, uint32_t k, uint32_t stream) {
    uint32_t h = sph_mix32(seed ^ 0x9e3779b9u);
    h = sph_mix32(h ^ counter);
    h = sph_mix32(h ^ ((slot << 2) | stream));
    h = sph_mix32(h ^ id);
    return sph_mix32(h ^ k);
}

// [0, 1): the top 24 bits times 2^-24, exact in float32
SPH_HD float sph_hash_unit(uint32_t h) { return (float)(h >> 8) * (1.0f / 16777216.0f); }
