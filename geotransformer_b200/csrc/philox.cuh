// Counter-based Philox4x32-10 shared by the correspondence RANSAC (ransac.cu) and the ground-truth superpoint target sampler
// (train.cu): a draw depends on (key, counter) only, never on the launch geometry or the rest of the batch.
#pragma once
#include <stdint.h>

namespace geob200 {

// Philox4x32-10 (Salmon et al., SC'11; the generator of curand_philox4x32_10): counter c, key (k0, k1), 10 rounds
__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
        const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
    }
}

}  // namespace geob200
