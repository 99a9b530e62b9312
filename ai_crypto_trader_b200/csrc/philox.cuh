// Philox4x32-10 counter-based RNG (Salmon et al., SC'11), shared by the Monte-Carlo kernels and the GA operators.
#pragma once
#include <stdint.h>

namespace b200bt {

struct Philox {
    uint32_t k0, k1;
};

__host__ __device__ __forceinline__ void philox_round(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3,
                                                      uint32_t k0, uint32_t k1) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    const uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}

// Philox4x32-10 (Salmon et al., SC'11): counter (c0..c3), key (k0,k1).
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                       uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        philox_round(c0, c1, c2, c3, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// One Philox block of Monte-Carlo path p: key = seed, counter words 0 and 1 = the global path index path_offset + p, so a
// path does not depend on the launch geometry or on how the paths are sharded.  Words 2 and 3 are the caller's.
__device__ __forceinline__ void philox_path(uint64_t seed, uint64_t path_offset, int64_t p, uint32_t c2, uint32_t c3,
                                            uint32_t out[4]) {
    const uint64_t gid = path_offset + (uint64_t)p;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    const uint32_t c0 = (uint32_t)gid, c1 = (uint32_t)(gid >> 32);
    philox4x32_10(c0, c1, c2, c3, k0, k1, out);
}

// Circular block bootstrap over a table of R entries, one index per random word u: a block starts at the uniform index
// __umulhi(u, R) and continues with the next entries, wrapping at R, for block_len draws.  Words drawn inside a block
// are not used.  The single-asset, joint and trade bootstraps all draw through this, so their index streams agree.
struct BlockBootstrap {
    int idx = 0, left = 0;
    __device__ __forceinline__ int next(uint32_t u, int R, int block_len) {
        if (left == 0) {
            idx = (int)__umulhi(u, (uint32_t)R);
            left = block_len;
        } else {
            idx = idx + 1 == R ? 0 : idx + 1;
        }
        --left;
        return idx;
    }
};

}  // namespace b200bt
