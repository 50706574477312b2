// Point-to-node grouping (superpoint patches) and k-NN partition.
//
// Reference: geotransformer/modules/ops/pointcloud_partition.py:35-107 (knn_partition, point_to_node_partition),
// with squared distances in the matmul form of ops/pairwise_distance.py:20-30:
//     d2 = clamp( |x|^2 - 2 x.y + |y|^2 , 0 )
// (NOT (x-y)^2: the argmin / top-k indices downstream depend on this rounding).
// The reference materialises an (M,N) distance matrix, a boolean (M,N) mask and runs a full top-k over N per node;
// here each point finds its node in one pass and each node sorts only its own points in shared memory.
#include "common.cuh"
#include "geob200.h"

namespace geob200 {

__device__ __forceinline__ float sqdist_mm(float ax, float ay, float az, float a2, float bx, float by, float bz, float b2) {
    // xy accumulated like a K=3 GEMM inner product with fused multiply-adds
    const float xy = fmaf(az, bz, fmaf(ay, by, __fmul_rn(ax, bx)));
    const float d = __fadd_rn(__fsub_rn(a2, __fmul_rn(2.0f, xy)), b2);
    return fmaxf(d, 0.0f);
}
__device__ __forceinline__ float sqnorm3(float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}

// argmin over nodes for every point; node occupancy flags.  Cloud s = blockIdx.y: points at Pt.start[s], nodes at Nd.start[s]
// (indices local to the cloud).
__global__ void __launch_bounds__(256) p2n_assign_kernel(const float* __restrict__ pts, const float* __restrict__ nodes,
                                                         const __grid_constant__ Segs Pt, const __grid_constant__ Segs Nd,
                                                         long long* __restrict__ point_to_node,
                                                         unsigned char* __restrict__ node_masks, int* __restrict__ node_count) {
    extern __shared__ float4 nd[];   // (x,y,z,|n|^2)
    const int s = blockIdx.y;
    const int N = Pt.count[s], M = Nd.count[s];
    if ((int)blockIdx.x * (int)blockDim.x >= N) return;
    pts += 3ll * Pt.start[s]; point_to_node += Pt.start[s];
    nodes += 3ll * Nd.start[s]; node_masks += Nd.start[s]; node_count += Nd.start[s];
    for (int m = threadIdx.x; m < M; m += blockDim.x) {
        const float x = nodes[3 * m], y = nodes[3 * m + 1], z = nodes[3 * m + 2];
        nd[m] = make_float4(x, y, z, sqnorm3(x, y, z));
    }
    __syncthreads();
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float px = pts[3ll * n], py = pts[3ll * n + 1], pz = pts[3ll * n + 2];
    const float p2 = sqnorm3(px, py, pz);
    float best = INFINITY;
    int bi = 0;
    for (int m = 0; m < M; ++m) {
        const float4 q = nd[m];
        const float d = sqdist_mm(q.x, q.y, q.z, q.w, px, py, pz, p2);
        if (d < best) { best = d; bi = m; }   // strict: first minimum wins, like torch.min
    }
    point_to_node[n] = bi;
    node_masks[bi] = 1;
    atomicAdd(&node_count[bi], 1);
}

// One CTA per node: the K nearest candidate points in ascending (d2, index) order.  Candidates = the node's own points
// (point_to_node != NULL: point_to_node_partition) or every point (NULL: knn_partition).  The point range is walked in chunks;
// candidates are appended to a shared-memory buffer of (d2 bits << 32 | index) keys which is bitonic-sorted and cut back to
// the best K whenever the next chunk might not fit, so any number of candidates is handled exactly (the former fixed 4096
// capacity is gone).  d2 in the reference's matmul form, node first: pairwise_distance(nodes, points).
// Cloud s = blockIdx.y: points (and point_to_node) at Pt.start[s], nodes and output rows at Nd.start[s].
template <int CAP>
__global__ void __launch_bounds__(256) knn_select_kernel(const float* __restrict__ pts, const float* __restrict__ nodes,
                                                         const __grid_constant__ Segs Pt, const __grid_constant__ Segs Nd,
                                                         const long long* __restrict__ point_to_node, int K,
                                                         long long* __restrict__ knn_indices, unsigned char* __restrict__ knn_masks,
                                                         float* __restrict__ knn_sqdist) {
    __shared__ unsigned long long keys[CAP];
    __shared__ int cnt;
    const int s = blockIdx.y;
    const int m = blockIdx.x;
    if (m >= Nd.count[s]) return;
    const int N = Pt.count[s];
    pts += 3ll * Pt.start[s];
    if (point_to_node != nullptr) point_to_node += Pt.start[s];
    nodes += 3ll * Nd.start[s];
    knn_indices += (long long)Nd.start[s] * K;
    if (knn_masks != nullptr) knn_masks += (long long)Nd.start[s] * K;
    if (knn_sqdist != nullptr) knn_sqdist += (long long)Nd.start[s] * K;
    const int CH = CAP - K;                       // a chunk can add at most CH candidates on top of the K kept ones
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const float nx = nodes[3 * m], ny = nodes[3 * m + 1], nz = nodes[3 * m + 2];
    const float n2 = sqnorm3(nx, ny, nz);
    for (int base = 0; base < N; base += CH) {
        const int end = min(N, base + CH);
        for (int n = base + threadIdx.x; n < end; n += blockDim.x) {
            if (point_to_node == nullptr || point_to_node[n] == m) {
                const float px = pts[3ll * n], py = pts[3ll * n + 1], pz = pts[3ll * n + 2];
                const float d = sqdist_mm(nx, ny, nz, n2, px, py, pz, sqnorm3(px, py, pz));
                const int pos = atomicAdd(&cnt, 1);
                keys[pos] = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)n;
            }
        }
        __syncthreads();
        const int c = cnt;
        __syncthreads();                          // every thread has read cnt before the next chunk's atomicAdd changes it
        const bool last = end >= N;
        if (!last && c + CH <= CAP) continue;     // the next chunk still fits: keep appending (uniform branch)
        int n2p = 1;
        while (n2p < c) n2p <<= 1;
        for (int i = c + threadIdx.x; i < n2p; i += blockDim.x) keys[i] = 0xFFFFFFFFFFFFFFFFull;
        __syncthreads();
        for (int k = 2; k <= n2p; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int t = threadIdx.x; t < n2p; t += blockDim.x) {
                    const int p = t ^ j;
                    if (p > t) {
                        const unsigned long long a = keys[t], b = keys[p];
                        const bool up = ((t & k) == 0);
                        if ((a > b) == up) { keys[t] = b; keys[p] = a; }
                    }
                }
                __syncthreads();
            }
        if (threadIdx.x == 0) cnt = min(c, K);
        __syncthreads();
    }
    const int c = cnt;
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        const bool ok = i < c;
        knn_indices[(long long)m * K + i] = ok ? (long long)(unsigned)(keys[i] & 0xFFFFFFFFull) : (long long)N;
        if (knn_masks != nullptr) knn_masks[(long long)m * K + i] = ok ? 1 : 0;
        if (knn_sqdist != nullptr) knn_sqdist[(long long)m * K + i] = ok ? __uint_as_float((unsigned)(keys[i] >> 32)) : INFINITY;
    }
}

// pairwise_distance (ops/pairwise_distance.py:4-31) for row-major (N, C) x (M, C): clamp(x2 - 2 xy + y2, 0), or 2 - 2 xy
__global__ void __launch_bounds__(256) pairwise_distance_kernel(const float* __restrict__ x, int N, const float* __restrict__ y, int M,
                                                                int C, int normalized, float* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)N * M) return;
    const int i = (int)(t / M), j = (int)(t % M);
    const float* a = x + (long long)i * C;
    const float* b = y + (long long)j * C;
    float xy = 0.f, a2 = 0.f, b2 = 0.f;
    for (int c = 0; c < C; ++c) {
        const float u = a[c], v = b[c];
        xy = (c == 0) ? __fmul_rn(u, v) : fmaf(u, v, xy);
        a2 = __fadd_rn(a2, __fmul_rn(u, u));
        b2 = __fadd_rn(b2, __fmul_rn(v, v));
    }
    const float d = normalized ? __fsub_rn(2.0f, __fmul_rn(2.0f, xy)) : __fadd_rn(__fsub_rn(a2, __fmul_rn(2.0f, xy)), b2);
    out[t] = fmaxf(d, 0.0f);
}

// get_point_to_node_indices (pointcloud_partition.py:9-32): argmin over nodes of pairwise_distance(points, nodes), i.e. the
// POINT-first rounding (p2 - 2xy) + n2 (point_to_node_partition uses the node-first one)
__global__ void __launch_bounds__(256) p2n_indices_kernel(const float* __restrict__ pts, int N, const float* __restrict__ nodes, int M,
                                                          long long* __restrict__ indices, int* __restrict__ node_count) {
    extern __shared__ float4 nd[];
    for (int m = threadIdx.x; m < M; m += blockDim.x) {
        const float x = nodes[3 * m], y = nodes[3 * m + 1], z = nodes[3 * m + 2];
        nd[m] = make_float4(x, y, z, sqnorm3(x, y, z));
    }
    __syncthreads();
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float px = pts[3ll * n], py = pts[3ll * n + 1], pz = pts[3ll * n + 2];
    const float p2 = sqnorm3(px, py, pz);
    float best = INFINITY;
    int bi = 0;
    for (int m = 0; m < M; ++m) {
        const float4 q = nd[m];
        const float d = sqdist_mm(px, py, pz, p2, q.x, q.y, q.z, q.w);
        if (d < best) { best = d; bi = m; }
    }
    indices[n] = bi;
    if (node_count != nullptr) atomicAdd(&node_count[bi], 1);
}

// apply_transform (ops/transformation.py:7-60): out = P R^T + t for one 4x4 transform (device pointer)
__global__ void __launch_bounds__(256) apply_transform_kernel(const float* __restrict__ pts, long long n, const float* __restrict__ T,
                                                              float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        out[3 * i + r] = __fadd_rn(fmaf(z, T[4 * r + 2], fmaf(y, T[4 * r + 1], __fmul_rn(x, T[4 * r]))), T[4 * r + 3]);
}

// gather rows of a zero-padded table: out[r] = (idx[r] < n_rows) ? table[idx[r]] : 0   (index_select on padded tables,
// EXP*/model.py:105-108,169-180)
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ table, int n_rows, int C,
                                                          const long long* __restrict__ idx, long long n_idx,
                                                          float* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_idx * C) return;
    const long long r = t / C;
    const int c = (int)(t % C);
    const long long i = idx[r];
    out[t] = (i >= 0 && i < n_rows) ? table[i * C + c] : 0.f;
}

}  // namespace geob200

using namespace geob200;

extern "C" {

int geob200_point_to_node_partition_batched(const float* points, const float* nodes, int64_t n_clouds, const int64_t* cloud_points,
                                            const int64_t* cloud_nodes, int64_t point_limit, int64_t* point_to_node, uint8_t* node_masks,
                                            int32_t* node_sizes, int64_t* node_knn_indices, uint8_t* node_knn_masks, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    Segs Pt, Nd;
    if (segs_from_counts(&Pt, n_clouds, cloud_points) || segs_from_counts(&Nd, n_clouds, cloud_nodes)) return -1;
    GEOB_REQUIRE(Pt.max > 0 && Nd.max > 0, "point_to_node_partition: empty input");
    GEOB_REQUIRE(point_limit > 0 && point_limit <= 2048, "point_to_node_partition: point_limit must be in 1..2048 (got %lld)",
                 (long long)point_limit);
    GEOB_REQUIRE((int64_t)Nd.max * 16 <= 200 * 1024, "point_to_node_partition: too many nodes (%d)", Nd.max);
    const int64_t n_nodes = (int64_t)Nd.start[n_clouds - 1] + Nd.count[n_clouds - 1];
    GEOB_CHECK_CUDA(cudaMemsetAsync(node_masks, 0, n_nodes, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(node_sizes, 0, 4 * n_nodes, st));
    const size_t smem = sizeof(float4) * Nd.max;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)p2n_assign_kernel)) return -1;
    p2n_assign_kernel<<<dim3((unsigned)((Pt.max + 255) / 256), Pt.n), 256, smem, st>>>(points, nodes, Pt, Nd, (long long*)point_to_node,
                                                                                     node_masks, node_sizes);
    knn_select_kernel<4096><<<dim3((unsigned)Nd.max, Nd.n), 256, 0, st>>>(points, nodes, Pt, Nd, (const long long*)point_to_node,
                                                                         (int)point_limit, (long long*)node_knn_indices, node_knn_masks, nullptr);
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

int geob200_knn_partition(const float* points, int64_t n_points, const float* nodes, int64_t n_nodes, int64_t k,
                          int64_t* knn_indices, float* knn_sq_distances, void* stream) {
    GEOB_REQUIRE(n_points > 0 && n_nodes > 0 && k > 0 && k <= n_points, "knn_partition: need 0 < k <= n_points");
    GEOB_REQUIRE(k <= 2048, "knn_partition: k <= 2048 supported (got %lld)", (long long)k);
    knn_select_kernel<4096><<<dim3((unsigned)n_nodes, 1), 256, 0, (cudaStream_t)stream>>>(points, nodes, segs_one(n_points), segs_one(n_nodes),
                                                                                         nullptr, (int)k, (long long*)knn_indices, nullptr,
                                                                                         knn_sq_distances);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_pairwise_distance(const float* x, int64_t n, const float* y, int64_t m, int64_t channels, int normalized, float* out,
                              void* stream) {
    if (n == 0 || m == 0) return 0;
    GEOB_REQUIRE(channels > 0, "pairwise_distance: channels must be positive");
    const long long total = n * m;
    pairwise_distance_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, (int)n, y, (int)m, (int)channels,
                                                                                              normalized, out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_point_to_node_indices(const float* points, int64_t n_points, const float* nodes, int64_t n_nodes, int64_t* indices,
                                  int32_t* node_sizes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_points > 0 && n_nodes > 0, "get_point_to_node_indices: empty input");
    GEOB_REQUIRE(n_nodes * 16 <= 48 * 1024, "get_point_to_node_indices: too many nodes (%lld)", (long long)n_nodes);
    if (node_sizes != nullptr) GEOB_CHECK_CUDA(cudaMemsetAsync(node_sizes, 0, 4 * n_nodes, st));
    p2n_indices_kernel<<<(unsigned)((n_points + 255) / 256), 256, sizeof(float4) * n_nodes, st>>>(points, (int)n_points, nodes,
                                                                                                  (int)n_nodes, (long long*)indices, node_sizes);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_apply_transform(const float* points, int64_t n_points, const float* transform, float* out, void* stream) {
    if (n_points == 0) return 0;
    apply_transform_kernel<<<(unsigned)((n_points + 255) / 256), 256, 0, (cudaStream_t)stream>>>(points, n_points, transform, out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_gather_rows(const float* table, int64_t n_rows, int64_t channels, const int64_t* indices, int64_t n_indices,
                        float* out, void* stream) {
    if (n_indices == 0) return 0;
    const long long total = n_indices * channels;
    gather_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(table, (int)n_rows, (int)channels,
                                                                                        (const long long*)indices, n_indices, out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
