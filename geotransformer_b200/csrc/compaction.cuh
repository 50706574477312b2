// Ordered in-CTA compaction shared by the ground-truth superpoint target sampler (train.cu) and the training-data augmentation
// (augment.cu).
#pragma once
#include "common.cuh"

namespace geob200 {

// Ordered compaction of one CTA-wide chunk (WARPS x 32 threads, the whole CTA): flag of this thread -> its rank among the flagged
// threads of the chunk (in thread order); *chunk_total receives the chunk's count.  warp_tot: WARPS shared words.
template <int WARPS = 32>
__device__ __forceinline__ int chunk_rank(bool flag, int* warp_tot, int* chunk_total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    int off = __popc(bal & ((1u << lane) - 1u)), tot = 0;
    for (int w = 0; w < WARPS; ++w) {
        const int c = warp_tot[w];
        off += w < warp ? c : 0;
        tot += c;
    }
    __syncthreads();                       // warp_tot is reused by the next chunk
    *chunk_total = tot;
    return off;
}

}  // namespace geob200
