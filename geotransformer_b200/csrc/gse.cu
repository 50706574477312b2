// Geometric structure embedding (pair-wise distance + triplet-wise angle embedding).
//
// Reference: geotransformer/modules/geotransformer/geotransformer.py:27-72 and
//            geotransformer/modules/transformer/positional_embedding.py:8-34.
//   E[i,j,:] = proj_d(sinus(d_ij / sigma_d)) + max_k proj_a(sinus(angle_ijk * 180/(sigma_a*pi)))
// The reference materialises two (N,N,{1,3},C) sinusoid tensors in HBM (0.45 GB at N=271,C=256) and runs
// (N^2*4, C) x (C, C) GEMMs over them.  Here the sinusoid tile is generated on chip, contracted, and only
// E (N,N,C) is written: the O(N^2 k C) intermediate never exists.
//
// This file holds the index kernel and the fp32 CUDA-core contraction (exact-fp32 reference path).  The
// wgmma tensor-core contraction lives in gse_tc.cu and is selected by geob200_structure_embedding().
#include "common.cuh"
#include "geob200.h"

namespace geob200 {

__device__ __forceinline__ float sqnorm3g(float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}
__device__ __forceinline__ float dist_mm(float ax, float ay, float az, float a2, float bx, float by, float bz, float b2) {
    const float xy = fmaf(az, bz, fmaf(ay, by, __fmul_rn(ax, bx)));
    return sqrtf(fmaxf(__fadd_rn(__fsub_rn(a2, __fmul_rn(2.0f, xy)), b2), 0.0f));   // sqrt(pairwise_distance)
}

// One warp per anchor point i: distances to every j, the (k+1) nearest (the first is dropped, geotransformer.py:42),
// then the k triplet angles for every j.  d_idx (N,N), a_idx (N,N,KA).
// Clouds of a batch (blockIdx.y = cloud): stacked points, d / a outputs concatenated cloud after cloud (cloud c at pair_start[c]).
struct GseClouds {
    int n_clouds;
    int row_start[GEOB_MAX_CLOUDS + 1];
    long long pair_start[GEOB_MAX_CLOUDS + 1];
};

template <int KA>
__global__ void __launch_bounds__(256) gse_indices_kernel(const float* __restrict__ pts_all, int N_single, float sigma_d, float factor_a,
                                                          float* __restrict__ d_all, float* __restrict__ a_all,
                                                          const __grid_constant__ GseClouds cl) {
    extern __shared__ float4 ps[];     // (x,y,z,|p|^2)
    // single cloud (n_clouds == 0): the arguments describe it; batch: cloud blockIdx.y of the descriptor
    const int cloud = blockIdx.y;
    const int N = cl.n_clouds > 0 ? cl.row_start[cloud + 1] - cl.row_start[cloud] : N_single;
    const float* __restrict__ pts = cl.n_clouds > 0 ? pts_all + 3ll * cl.row_start[cloud] : pts_all;
    float* __restrict__ d_idx = cl.n_clouds > 0 ? d_all + cl.pair_start[cloud] : d_all;
    float* __restrict__ a_idx = cl.n_clouds > 0 ? a_all + cl.pair_start[cloud] * KA : a_all;
    if ((int)(blockIdx.x * (blockDim.x >> 5)) >= N) return;          // grid.x covers the largest cloud
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
        const float x = pts[3 * n], y = pts[3 * n + 1], z = pts[3 * n + 2];
        ps[n] = make_float4(x, y, z, sqnorm3g(x, y, z));
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= N) return;
    const float4 pi = ps[i];
    for (int j = lane; j < N; j += 32) {
        const float4 pj = ps[j];
        d_idx[(long long)i * N + j] = dist_mm(pi.x, pi.y, pi.z, pi.w, pj.x, pj.y, pj.z, pj.w) / sigma_d;
    }
    // (KA+1) smallest by (distance, index); selection rounds with a strictly increasing key
    unsigned long long last = 0;
    bool first = true;
    int knn[KA];
#pragma unroll
    for (int r = 0; r <= KA; ++r) {
        unsigned long long best = 0xFFFFFFFFFFFFFFFFull;
        for (int j = lane; j < N; j += 32) {
            const float4 pj = ps[j];
            const float d = dist_mm(pi.x, pi.y, pi.z, pi.w, pj.x, pj.y, pj.z, pj.w);
            const unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)j;
            if ((first || key > last) && key < best) best = key;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
            best = other < best ? other : best;
        }
        last = best;
        first = false;
        if (r > 0) knn[r - 1] = (int)(best & 0xFFFFFFFFull);
    }
    float rx[KA], ry[KA], rz[KA];
#pragma unroll
    for (int k = 0; k < KA; ++k) {
        // fewer than KA+1 points: best stays at the all-ones key; clamp (the reference would raise in topk)
        const int kk = min(knn[k], N - 1);
        const float4 pk = ps[kk];
        rx[k] = pk.x - pi.x; ry[k] = pk.y - pi.y; rz[k] = pk.z - pi.z;      // ref_vectors = p_knn - p_i
    }
    for (int j = lane; j < N; j += 32) {
        const float4 pj = ps[j];
        const float ax = pj.x - pi.x, ay = pj.y - pi.y, az = pj.z - pi.z;  // anc_vectors = p_j - p_i
#pragma unroll
        for (int k = 0; k < KA; ++k) {
            const float cx = __fsub_rn(__fmul_rn(ry[k], az), __fmul_rn(rz[k], ay));
            const float cy = __fsub_rn(__fmul_rn(rz[k], ax), __fmul_rn(rx[k], az));
            const float cz = __fsub_rn(__fmul_rn(rx[k], ay), __fmul_rn(ry[k], ax));
            const float sinv = sqrtf(sqnorm3g(cx, cy, cz));
            // accumulate from +0 like torch.sum: a sum of negative zeros (j == i) must give +0 so that atan2(0, 0) = 0, not pi
            const float cosv = __fadd_rn(__fadd_rn(__fadd_rn(0.0f, __fmul_rn(rx[k], ax)), __fmul_rn(ry[k], ay)), __fmul_rn(rz[k], az));
            a_idx[((long long)i * N + j) * KA + k] = atan2f(sinv, cosv) * factor_a;
        }
    }
}

// ---- fp32 contraction ------------------------------------------------------------------------------------
// CTA tile: 32 (i,j) pairs = 128 sinusoid rows (d, a0, a1, a2) x C=256 outputs, K = 256 in chunks of 16.
// A (sinusoids) is generated once into shared memory; WdT / WaT ((in, out) = transposed nn.Linear weights) are
// streamed through shared memory.  Each thread owns 2 pairs x 4 sub-rows x 16 columns.
constexpr int GSE_C = 256;
constexpr int GSE_PAIRS = 32;
constexpr int GSE_AST = GSE_C + 4;
constexpr int GSE_BK = 16;

__global__ void __launch_bounds__(256, 1) gse_embed_fp32_kernel(const float* __restrict__ d_idx, const float* __restrict__ a_idx,
                                                                long long n_pairs, const float* __restrict__ div_term,
                                                                const float* __restrict__ WdT, const float* __restrict__ WaT,
                                                                const float* __restrict__ bd, const float* __restrict__ ba,
                                                                float* __restrict__ E) {
    extern __shared__ float sm[];
    float* A = sm;                                    // [4][32][AST]
    float* Bd = A + 4 * GSE_PAIRS * GSE_AST;          // [BK][256]
    float* Ba = Bd + GSE_BK * GSE_C;                  // [BK][256]
    const long long p0 = (long long)blockIdx.x * GSE_PAIRS;
    {
        // generate sinusoids: thread -> (row = t>>1 in [0,128), half of the 128 frequencies)
        const int row = threadIdx.x >> 1, half = threadIdx.x & 1;
        const int s = row >> 5, pr = row & 31;
        const long long p = p0 + pr;
        float x = 0.f;
        if (p < n_pairs) x = (s == 0) ? d_idx[p] : a_idx[p * 3 + (s - 1)];
        float* arow = A + (s * GSE_PAIRS + pr) * GSE_AST;
        for (int f = half * 64; f < half * 64 + 64; ++f) {
            float sv, cv;
            sincosf(__fmul_rn(x, div_term[f]), &sv, &cv);
            *reinterpret_cast<float2*>(arow + 2 * f) = make_float2(sv, cv);   // interleaved [sin, cos]
        }
    }
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[2][4][16];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int c = 0; c < 16; ++c) acc[a][s][c] = 0.f;

    for (int k0 = 0; k0 < GSE_C; k0 += GSE_BK) {
        __syncthreads();
        for (int e = threadIdx.x; e < GSE_BK * GSE_C / 4; e += 256) {
            reinterpret_cast<float4*>(Bd)[e] = reinterpret_cast<const float4*>(WdT + (long long)k0 * GSE_C)[e];
            reinterpret_cast<float4*>(Ba)[e] = reinterpret_cast<const float4*>(WaT + (long long)k0 * GSE_C)[e];
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < GSE_BK; kk += 4) {
            float4 av[2][4];
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int s = 0; s < 4; ++s)
                    av[a][s] = *reinterpret_cast<const float4*>(A + (s * GSE_PAIRS + ty + 16 * a) * GSE_AST + k0 + kk);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float4 bdv[4], bav[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    bdv[j] = *reinterpret_cast<const float4*>(Bd + (kk + u) * GSE_C + tx * 4 + 64 * j);
                    bav[j] = *reinterpret_cast<const float4*>(Ba + (kk + u) * GSE_C + tx * 4 + 64 * j);
                }
#pragma unroll
                for (int a = 0; a < 2; ++a) {
#pragma unroll
                    for (int s = 0; s < 4; ++s) {
                        const float4 v4 = av[a][s];
                        const float xa = (u == 0) ? v4.x : (u == 1) ? v4.y : (u == 2) ? v4.z : v4.w;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float4 b = (s == 0) ? bdv[j] : bav[j];
                            acc[a][s][4 * j + 0] = fmaf(xa, b.x, acc[a][s][4 * j + 0]);
                            acc[a][s][4 * j + 1] = fmaf(xa, b.y, acc[a][s][4 * j + 1]);
                            acc[a][s][4 * j + 2] = fmaf(xa, b.z, acc[a][s][4 * j + 2]);
                            acc[a][s][4 * j + 3] = fmaf(xa, b.w, acc[a][s][4 * j + 3]);
                        }
                    }
                }
            }
        }
    }
    // epilogue: E = (acc_d + bd) + max_k (acc_ak + ba)
#pragma unroll
    for (int a = 0; a < 2; ++a) {
        const long long p = p0 + ty + 16 * a;
        if (p >= n_pairs) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = tx * 4 + 64 * j;
            const float4 bdv = *reinterpret_cast<const float4*>(bd + c);
            const float4 bav = *reinterpret_cast<const float4*>(ba + c);
            float o[4];
            const float bdd[4] = {bdv.x, bdv.y, bdv.z, bdv.w}, baa[4] = {bav.x, bav.y, bav.z, bav.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float m = fmaxf(fmaxf(acc[a][1][4 * j + u] + baa[u], acc[a][2][4 * j + u] + baa[u]), acc[a][3][4 * j + u] + baa[u]);
                o[u] = (acc[a][0][4 * j + u] + bdd[u]) + m;
            }
            *reinterpret_cast<float4*>(E + p * GSE_C + c) = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
}

// Generic (any C multiple of 4, e.g. KITTI hidden_dim 128) fp32 contraction, one warp per pair; slower, used when
// C != 256.  out channel c handled by lane-strided loop; sinusoid rows staged per warp in shared memory.
__global__ void __launch_bounds__(256) gse_embed_generic_kernel(const float* __restrict__ d_idx, const float* __restrict__ a_idx,
                                                                long long n_pairs, int C, const float* __restrict__ div_term,
                                                                const float* __restrict__ WdT, const float* __restrict__ WaT,
                                                                const float* __restrict__ bd, const float* __restrict__ ba,
                                                                float* __restrict__ E) {
    extern __shared__ float sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* A = sm + warp * 4 * C;      // [4][C]
    const long long p = (long long)blockIdx.x * 8 + warp;
    if (p >= n_pairs) return;
    float x[4] = {d_idx[p], a_idx[p * 3], a_idx[p * 3 + 1], a_idx[p * 3 + 2]};
    for (int f = lane; f < C / 2; f += 32) {
        const float dv = div_term[f];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            float sv, cv;
            sincosf(__fmul_rn(x[s], dv), &sv, &cv);
            A[s * C + 2 * f] = sv;
            A[s * C + 2 * f + 1] = cv;
        }
    }
    __syncwarp();
    for (int c = lane; c < C; c += 32) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int k = 0; k < C; ++k) {
            const float wd = WdT[(long long)k * C + c], wa = WaT[(long long)k * C + c];
            a0 = fmaf(A[k], wd, a0);
            a1 = fmaf(A[C + k], wa, a1);
            a2 = fmaf(A[2 * C + k], wa, a2);
            a3 = fmaf(A[3 * C + k], wa, a3);
        }
        const float m = fmaxf(fmaxf(a1 + ba[c], a2 + ba[c]), a3 + ba[c]);
        E[p * C + c] = (a0 + bd[c]) + m;
    }
}

}  // namespace geob200

using namespace geob200;

// implemented in gse_tc.cu (wgmma tensor-core contraction); returns 1 if it does not handle this shape/mode
int geob200_gse_embed_tc(const float* d_idx, const float* a_idx, long long n_pairs, int C, const float* div_term,
                         const float* Wd, const float* Wa, const float* bd, const float* ba, float* E, int mode,
                         void* workspace, size_t workspace_bytes, cudaStream_t st);

extern "C" {

int geob200_gse_indices(const float* points, int64_t n, float sigma_d, float factor_a, int64_t angle_k, float* d_indices,
                        float* a_indices, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n > 0, "gse_indices: empty cloud");
    GEOB_REQUIRE(angle_k == 3, "gse_indices: angle_k=%lld unsupported (all shipped models use 3)", (long long)angle_k);
    GEOB_REQUIRE(n * 16 <= 200 * 1024, "gse_indices: too many superpoints (%lld)", (long long)n);
    const size_t smem = sizeof(float4) * n;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)gse_indices_kernel<3>)) return -1;
    GseClouds none{};
    gse_indices_kernel<3><<<(unsigned)((n + 7) / 8), 256, smem, st>>>(points, (int)n, sigma_d, factor_a, d_indices, a_indices, none);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_gse_indices_batched(const float* points, int64_t n_clouds, const int64_t* cloud_rows_h, float sigma_d, float factor_a,
                                int64_t angle_k, float* d_indices, float* a_indices, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_clouds >= 1 && n_clouds <= GEOB_MAX_CLOUDS, "gse_indices: 1..%d clouds per launch", GEOB_MAX_CLOUDS);
    GEOB_REQUIRE(angle_k == 3, "gse_indices: angle_k=%lld unsupported (all shipped models use 3)", (long long)angle_k);
    GseClouds cl{};
    cl.n_clouds = (int)n_clouds;
    int64_t max_n = 0;
    for (int64_t c = 0; c < n_clouds; ++c) {
        const int64_t n = cloud_rows_h[c];
        GEOB_REQUIRE(n > 0, "gse_indices: empty cloud");
        cl.row_start[c + 1] = cl.row_start[c] + (int)n;
        cl.pair_start[c + 1] = cl.pair_start[c] + n * n;
        max_n = n > max_n ? n : max_n;
    }
    GEOB_REQUIRE(max_n * 16 <= 200 * 1024, "gse_indices: too many superpoints (%lld)", (long long)max_n);
    const size_t smem = sizeof(float4) * max_n;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)gse_indices_kernel<3>)) return -1;
    const dim3 grid((unsigned)((max_n + 7) / 8), (unsigned)n_clouds);
    gse_indices_kernel<3><<<grid, 256, smem, st>>>(points, 0, sigma_d, factor_a, d_indices, a_indices, cl);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

size_t geob200_gse_embed_workspace_bytes(int64_t n, int64_t channels) {
    (void)n;
    return (size_t)(4 * channels * channels * 4 * 3 + 4096);   // room for split/packed weight copies of the tensor-core path
}

// mode: 0 = fp32 CUDA cores (exact-fp32 accumulation), 1 = wgmma 3xTF32 (fp32-accurate), 2 = wgmma 1xTF32,
//       3 = wgmma 3xFP16 (fp32-accurate, half the tensor-pipe time of 3xTF32; default)
int geob200_gse_embed(const float* d_indices, const float* a_indices, int64_t n, int64_t channels, const float* div_term,
                      const float* wd_t, const float* wa_t, const float* wd, const float* wa, const float* bd, const float* ba,
                      float* embeddings, int mode, void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n > 0, "gse_embed: bad shape");
    return geob200_gse_embed_pairs(d_indices, a_indices, n * n, channels, div_term, wd_t, wa_t, wd, wa, bd, ba, embeddings, mode, workspace,
                                   workspace_bytes, stream);
}

int geob200_gse_embed_pairs(const float* d_indices, const float* a_indices, int64_t n_rows, int64_t channels, const float* div_term,
                            const float* wd_t, const float* wa_t, const float* wd, const float* wa, const float* bd, const float* ba,
                            float* embeddings, int mode, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_rows > 0 && channels > 0 && channels % 4 == 0, "gse_embed: bad shape");
    const long long n_pairs = (long long)n_rows;
    if (mode != 0) {
        int rc = geob200_gse_embed_tc(d_indices, a_indices, n_pairs, (int)channels, div_term, wd, wa, bd, ba, embeddings, mode,
                                      workspace, workspace_bytes, st);
        if (rc <= 0) return rc;
        GEOB_REQUIRE(false, "gse_embed: tensor-core mode %d does not support C=%lld (C = 256: modes 1-4, C = 128: mode 3)", mode,
                     (long long)channels);
    }
    if (channels == GSE_C) {
        const size_t smem = sizeof(float) * (4 * GSE_PAIRS * GSE_AST + 2 * GSE_BK * GSE_C);
        if (ensure_max_smem((const void*)gse_embed_fp32_kernel)) return -1;
        gse_embed_fp32_kernel<<<(unsigned)((n_pairs + GSE_PAIRS - 1) / GSE_PAIRS), 256, smem, st>>>(
            d_indices, a_indices, n_pairs, div_term, wd_t, wa_t, bd, ba, embeddings);
    } else {
        const size_t smem = sizeof(float) * 8 * 4 * channels;
        GEOB_REQUIRE(smem <= 48 * 1024, "gse_embed: channels too large for the generic path");
        gse_embed_generic_kernel<<<(unsigned)((n_pairs + 7) / 8), 256, smem, st>>>(d_indices, a_indices, n_pairs, (int)channels,
                                                                                 div_term, wd_t, wa_t, bd, ba, embeddings);
    }
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
