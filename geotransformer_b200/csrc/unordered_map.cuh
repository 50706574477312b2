// Pieces of the stacked-cloud collate shared by grid subsampling (collate.cu) and voxel downsampling (voxel.cu).
#pragma once
#include "common.cuh"

namespace geob200 {

struct CloudSeg {      // one cloud of a stacked batch
    int start;         // first row in the stacked array
    int len;           // number of rows
};

// Per-cloud exclusive scan of an int array (one CTA of 1024 threads per cloud); defined in collate.cu.
__global__ void seg_exclusive_scan_kernel(const int* __restrict__ in, int* __restrict__ out, const CloudSeg* __restrict__ segs,
                                          int* __restrict__ total);

// slot hash of the open-addressing voxel tables
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

// libstdc++ _Prime_rehash_policy bucket counts (max load factor 1, growth factor 2, sparse prime list): the
// table is rehashed to kBuckets[p] right before element number kBuckets[p-1]+1 is inserted.
static __constant__ unsigned long long kBuckets[27] = {13ull, 29ull, 59ull, 127ull, 257ull, 541ull, 1109ull, 2357ull,
    5087ull, 10273ull, 20753ull, 42043ull, 85229ull, 172933ull, 351061ull, 712697ull, 1447153ull, 2938679ull,
    5967347ull, 12117689ull, 24607243ull, 49969847ull, 101473717ull, 206062531ull, 418451333ull, 849749479ull,
    1725587117ull};

// Iteration order of a default-constructed libstdc++ std::unordered_map filled by operator[] with m distinct keys whose
// bucket hashes are hash[0..m) (element e inserted e-th).  libstdc++ keeps one singly linked node list; a node whose bucket is
// empty goes to the FRONT of the list, otherwise to the front of its bucket's group, and a rehash re-inserts the nodes in current
// list order by the same rule.  Hence, after processing a sequence S with bucket count nb, the list is S sorted by (first
// position of the node's bucket in S, own position in S), both DESCENDING.  Each growth phase is evaluated in parallel as a rank
// computation:
//   new_pos(j) = #{elements whose bucket was activated later} + #{same-bucket elements that came later}.
// Called by every thread of a 1024-thread CTA; cur / nxt / A / lnk hold m ints and act / head / cnt hold nb <= 2.2 m + 13 ints
// each, all in global memory (L2 resident).  Returns the array (cur or nxt) that lists the elements head -> tail.
__device__ __forceinline__ const int* unordered_map_order(int m, const unsigned long long* __restrict__ hash, int* cur, int* nxt, int* A, int* lnk,
                                          int* act, int* head, int* cnt) {
    __shared__ int warp_tot[32];
    __shared__ int carry_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    for (int phase = 0; phase < 27; ++phase) {
        const int lo = (phase == 0) ? 0 : (int)kBuckets[phase - 1];
        if (lo >= m) break;
        const unsigned long long nb = kBuckets[phase];
        const int n = (nb < (unsigned long long)m) ? (int)nb : m;

        for (long long b = threadIdx.x; b < (long long)nb; b += blockDim.x) { act[b] = 0x7fffffff; head[b] = -1; cnt[b] = 0; }
        for (int j = threadIdx.x; j < n; j += blockDim.x) A[j] = 0;
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const int e = (j < lo) ? cur[j] : j;
            const int bk = (int)(hash[e] % nb);
            atomicMin(&act[bk], j);
            lnk[j] = atomicExch(&head[bk], j);
            atomicAdd(&cnt[bk], 1);
        }
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const int e = (j < lo) ? cur[j] : j;
            const int bk = (int)(hash[e] % nb);
            if (act[bk] == j) A[j] = cnt[bk];
        }
        __syncthreads();
        // suffix-exclusive scan of A over [0,n): S[j] = sum_{a>j} A[a]; done back to front in chunks.
        if (threadIdx.x == 0) carry_s = 0;
        __syncthreads();
        for (int base = 0; base < n; base += 1024) {
            const int r = base + threadIdx.x;        // reversed index
            const int j = n - 1 - r;
            const int v = (r < n) ? A[j] : 0;
            int x = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (lane == 31) warp_tot[warp] = x;
            __syncthreads();
            if (warp == 0) {
                int w = warp_tot[lane];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    int y = __shfl_up_sync(0xffffffffu, w, o);
                    if (lane >= o) w += y;
                }
                warp_tot[lane] = w;
            }
            __syncthreads();
            const int carry = carry_s;
            if (r < n) A[j] = carry + (warp > 0 ? warp_tot[warp - 1] : 0) + (x - v);
            __syncthreads();
            if (threadIdx.x == 1023) carry_s = carry + warp_tot[31];
            __syncthreads();
        }
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const int e = (j < lo) ? cur[j] : j;
            const int bk = (int)(hash[e] % nb);
            int later = 0;
            for (int q = head[bk]; q >= 0; q = lnk[q]) later += (q > j);
            nxt[A[act[bk]] + later] = e;
        }
        __syncthreads();
        int* t = cur; cur = nxt; nxt = t;
    }
    return cur;
}

}  // namespace geob200
