// Block-wide selection of the k largest 32-bit keys, shared by the coarse top-k of the superpoint matching (matching.cu) and
// the ground-truth superpoint target sampler (train.cu).
#pragma once
#include "common.cuh"

namespace geob200 {

// MSB-first 8-bit radix select over the keys key(t), t in [0, total), by the whole CTA (0 < k <= total): on return thr is the
// bit pattern of the k-th largest key and need_eq the number of keys equal to thr that belong to the k largest (the caller keeps
// the lowest indices among the ties).  hist: 256 counters in shared memory; prefix_s / kth_s: two shared words.
template <class Key>
__device__ __forceinline__ void radix_select_kth(long long total, int k, Key key, unsigned* hist, unsigned* prefix_s, unsigned* kth_s,
                                                 unsigned& thr, int& need_eq) {
    unsigned prefix = 0, mask = 0;
    int remaining = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (long long t = threadIdx.x; t < total; t += blockDim.x) {
            const unsigned b = key(t);
            if ((b & mask) == prefix) atomicAdd(&hist[(b >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int rem = remaining;
            int d = 255;
            for (; d > 0; --d) {
                if ((int)hist[d] >= rem) break;
                rem -= (int)hist[d];
            }
            *prefix_s = prefix | ((unsigned)d << shift);
            *kth_s = (unsigned)rem;
        }
        __syncthreads();
        prefix = *prefix_s;
        remaining = (int)*kth_s;
        mask |= (255u << shift);
        __syncthreads();
    }
    thr = prefix;
    need_eq = remaining;
}

}  // namespace geob200
