// Counter-based RNG shared by the device stages that draw their own random numbers (csrc/masking.cu, csrc/cycle.cu):
// Philox4x32-10 (Salmon et al. 2011), key = seed, counter = (element, stream, call counter).  A stage keeps
// (seed, call counter) in device memory and advances the counter on the stream, so a captured CUDA graph draws fresh
// numbers on every replay; each kind of draw uses its own `stream` id, so draws never share a counter.
#pragma once
#include <stdint.h>

namespace smk {

struct U4 { uint32_t x, y, z, w; };

__device__ __forceinline__ U4 philox(uint64_t seed, uint64_t ctr, uint32_t stream, uint32_t elem_hi, uint32_t elem_lo) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    U4 c{elem_lo, elem_hi, (uint32_t)ctr ^ (stream << 28), (uint32_t)(ctr >> 32)};
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = U4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c;
}

__device__ __forceinline__ float u01(uint32_t r) { return (float)(r >> 8) * (1.0f / 16777216.0f); }          // [0, 1)

}  // namespace smk
