// numpy's legacy generator (np.random.RandomState / np.random.seed) on the device: MT19937 with numpy's int seeding, its 53-bit
// doubles, the masked-rejection interval draw of permutation / shuffle, and the polar Gaussian with its one-value cache.
//
// Warp-uniform: all 32 lanes of one warp call every method with the same arguments and hold identical copies of the scalar state
// (position, Gaussian cache); the 624-word key lives in shared memory, and the warp shares the seeding writes and the twist.  Every
// draw is exact integer arithmetic or correctly rounded double arithmetic (no contraction), except `log` in gauss(), whose last
// bit may differ from the host libm's; the accept / reject decisions, and so the sequence of words consumed, do not depend on it.
#pragma once
#include <stdint.h>

namespace geob200 {

constexpr int MT_N = 624, MT_M = 397;

struct LegacyRandom {
    uint32_t* key;                         // shared, MT_N words
    int pos;
    bool has_gauss;
    double gauss;

    // np.random.seed(s) for an integer 0 <= s < 2^32: key[0] = s, key[i] = 1812433253 (key[i-1] ^ (key[i-1] >> 30)) + i; the
    // Gaussian cache is cleared.  A serial recurrence: every lane runs it and writes its own stripe.
    __device__ __forceinline__ void seed(uint32_t s) {
        const int lane = threadIdx.x & 31;
        for (int i = 0; i < MT_N; ++i) {
            if ((i & 31) == lane) key[i] = s;
            s = 1812433253u * (s ^ (s >> 30)) + (uint32_t)(i + 1);
        }
        pos = MT_N;
        has_gauss = false;
        gauss = 0.0;
        __syncwarp();
    }

    // the 624-word regeneration, 32 words at a time in index order: word i reads words i + 1 and i + 397 (mod 624), which the
    // sequential loop has updated exactly when they precede i, i.e. in an earlier chunk (every read index is 227 or more before i
    // or after the chunk), so each chunk reads, then writes
    __device__ __forceinline__ void twist() {
        const int lane = threadIdx.x & 31;
        for (int base = 0; base < MT_N; base += 32) {
            const int i = base + lane;
            uint32_t v = 0;
            if (i < MT_N) {
                const uint32_t y = (key[i] & 0x80000000u) | (key[i + 1 < MT_N ? i + 1 : 0] & 0x7fffffffu);
                v = key[i + MT_M < MT_N ? i + MT_M : i + MT_M - MT_N] ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
            }
            __syncwarp();
            if (i < MT_N) key[i] = v;
            __syncwarp();
        }
        pos = 0;
    }

    __device__ __forceinline__ uint32_t next32() {
        if (pos == MT_N) twist();
        uint32_t y = key[pos++];
        y ^= y >> 11;
        y ^= (y << 7) & 0x9d2c5680u;
        y ^= (y << 15) & 0xefc60000u;
        y ^= y >> 18;
        return y;
    }

    // random_sample / rand: ((a >> 5) 2^26 + (b >> 6)) 2^-53, exact
    __device__ __forceinline__ double next_double() {
        const uint32_t a = next32() >> 5, b = next32() >> 6;
        return __dmul_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)b), 0x1p-53);
    }

    // uniform(low, high): low + (high - low) u
    __device__ __forceinline__ double uniform(double low, double high) { return __dadd_rn(low, __dmul_rn(__dsub_rn(high, low), next_double())); }

    // random_interval(max), max < 2^32: the low bits under the smallest all-ones mask covering max, rejected while > max
    __device__ __forceinline__ uint32_t interval(uint32_t max) {
        if (max == 0) return 0;
        uint32_t mask = max;
        mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
        uint32_t v;
        do v = next32() & mask;
        while (v > max);
        return v;
    }

    // legacy_gauss: the polar method; a call without a cached value draws a pair, returns f x2 and caches f x1
    __device__ __forceinline__ double gauss_draw() {
        if (has_gauss) {
            has_gauss = false;
            const double g = gauss;
            gauss = 0.0;
            return g;
        }
        double x1, x2, r2;
        do {
            x1 = __dsub_rn(__dmul_rn(2.0, next_double()), 1.0);
            x2 = __dsub_rn(__dmul_rn(2.0, next_double()), 1.0);
            r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));
        } while (r2 >= 1.0 || r2 == 0.0);
        const double f = __dsqrt_rn(__ddiv_rn(__dmul_rn(-2.0, log(r2)), r2));
        gauss = __dmul_rn(f, x1);
        has_gauss = true;
        return __dmul_rn(f, x2);
    }
};

}  // namespace geob200
