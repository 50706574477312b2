// Correspondence RANSAC and the per-pair correspondence metrics of the benchmark evaluation.
//
// Reference: geotransformer/utils/open3d.py:169-198 (registration_with_ransac_from_correspondences: Open3D's
//            registration_ransac_based_on_correspondence, TransformationEstimationPointToPoint(False), no checkers,
//            RANSACConvergenceCriteria(I, I)) and geotransformer/utils/registration.py:133-155, 240-250
//            (evaluate_correspondences: inlier ratio, overlap, mean residual).
// Open3D runs the I hypotheses on the CPU, one pair at a time.  Here a CTA owns 32 hypotheses of one pair (pair = blockIdx.y):
// every warp builds and keeps 4 of them in registers while the pair's correspondences stream through shared-memory tiles;
// a second launch picks the winner of every pair in a fixed order.  Semantics (DESIGN.md section 3b):
//   * all I iterations run: the reference passes I as the confidence, Open3D clamps it to 1.0 and log(1 - 1) = -inf makes the
//     early-exit estimate +inf (or NaN for an all-inlier hypothesis), so the exit never fires;
//   * iteration i draws ransac_n indices with replacement from a counter-based Philox4x32-10: key = seed, counter =
//     (i, pair id, draw block, 0) with pair id = pair_base + p, index = umulhi(word, n) -- a pair's draws depend on
//     (seed, pair id, n) only, not on the rest of the batch or the launch geometry (Open3D's random stream is not reproduced);
//   * hypothesis = unweighted Kabsch over the drawn pairs in double (kabsch.cuh), stored as fp32 (R, t);
//   * inlier: ||R src + t - ref||^2 < tau^2 in pinned fp32 arithmetic (no contraction), inlier d^2 summed in double;
//   * winner: more inliers, then lower fp32 rmse, then lower iteration (Open3D merges its OpenMP threads in arbitrary order);
//     a best hypothesis without inliers, or n < ransac_n, gives Open3D's default result (identity, fitness 0, rmse 0).
#include "common.cuh"
#include "geob200.h"
#include "feature_match.cuh"
#include "kabsch.cuh"
#include "philox.cuh"

namespace geob200 {

constexpr int RS_WARPS = 8, RS_HPW = 4, RS_HPB = RS_WARPS * RS_HPW, RS_TILE = 1024, RS_MAX_N = 8;
constexpr int CM_THREADS = 256, CM_TILE = 1024;

// squared residual of one correspondence under (R | t) = h[0..11] (row-major 3x4), pinned: ((r0 x + r1 y) + r2 z) + t,
// then (dx^2 + dy^2) + dz^2, every operation rounded on its own
__device__ __forceinline__ float rs_residual2(const float* h, float x, float y, float z, float u, float v, float w) {
    const float ax = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(h[0], x), __fmul_rn(h[1], y)), __fmul_rn(h[2], z)), h[3]);
    const float ay = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(h[4], x), __fmul_rn(h[5], y)), __fmul_rn(h[6], z)), h[7]);
    const float az = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(h[8], x), __fmul_rn(h[9], y)), __fmul_rn(h[10], z)), h[11]);
    const float dx = __fsub_rn(ax, u), dy = __fsub_rn(ay, v), dz = __fsub_rn(az, w);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ int rs_count(const int* counts, int p, int cap) {
    return counts == nullptr ? cap : min(max(counts[p], 0), cap);
}

// Build + score.  Grid (ceil(I / 32), B), 256 threads.  Hypothesis h = blockIdx.x * 32 + warp * 4 + k.
__global__ void __launch_bounds__(RS_WARPS * 32) ransac_hypotheses_kernel(
        const float* __restrict__ ref, const float* __restrict__ src, int cap, const int* __restrict__ counts, float tau2, int rn,
        int I, uint32_t key0, uint32_t key1, uint32_t pair_base, float* __restrict__ hyp_rt /*[B][I][12]*/, int* __restrict__ hyp_cnt,
        float* __restrict__ hyp_rmse, float* __restrict__ rec_T /*[B][I][16] or null*/, int* __restrict__ rec_cnt,
        float* __restrict__ rec_rmse, int* __restrict__ rec_samples /*[B][I][8] or null*/) {
    __shared__ float tile[6][RS_TILE];                 // src x y z, ref x y z
    __shared__ float hs[RS_HPB][12];
    const int p = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = rs_count(counts, p, cap);
    ref += 3ll * p * cap; src += 3ll * p * cap;
    const bool live = n >= rn;                         // uniform over the CTA
    const int h0 = blockIdx.x * RS_HPB + warp * RS_HPW;

    if (lane < RS_HPW) {
        const int h = h0 + lane;
        float* o = hs[warp * RS_HPW + lane];
        int idx[RS_MAX_N];
#pragma unroll
        for (int j = 0; j < RS_MAX_N; ++j) idx[j] = -1;
        if (live && h < I) {
            uint32_t c[4];
#pragma unroll
            for (int j = 0; j < RS_MAX_N; ++j) {
                if (j % 4 == 0) { c[0] = (uint32_t)h; c[1] = pair_base + (uint32_t)p; c[2] = (uint32_t)(j / 4); c[3] = 0u; philox4x32_10(c, key0, key1); }
                if (j < rn) idx[j] = (int)__umulhi(c[j % 4], (uint32_t)n);
            }
            double cs[3] = {0, 0, 0}, cr[3] = {0, 0, 0};
#pragma unroll
            for (int j = 0; j < RS_MAX_N; ++j)
                if (j < rn)
                    for (int a = 0; a < 3; ++a) { cs[a] += (double)src[3 * idx[j] + a]; cr[a] += (double)ref[3 * idx[j] + a]; }
            for (int a = 0; a < 3; ++a) { cs[a] /= rn; cr[a] /= rn; }
            double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, R[9];
#pragma unroll
            for (int j = 0; j < RS_MAX_N; ++j)
                if (j < rn)
                    for (int a = 0; a < 3; ++a)
                        for (int b = 0; b < 3; ++b)
                            H[3 * a + b] += ((double)src[3 * idx[j] + a] - cs[a]) * ((double)ref[3 * idx[j] + b] - cr[b]);
            kabsch_rotation(H, R);
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) o[4 * i + j] = (float)R[3 * i + j];
                o[4 * i + 3] = (float)(cr[i] - (R[3 * i] * cs[0] + R[3 * i + 1] * cs[1] + R[3 * i + 2] * cs[2]));
            }
        } else {
            for (int e = 0; e < 12; ++e) o[e] = (e % 5 == 0) ? 1.f : 0.f;           // identity (R | 0)
        }
        if (rec_samples != nullptr && h < I)
            for (int j = 0; j < RS_MAX_N; ++j) rec_samples[((long long)p * I + h) * RS_MAX_N + j] = idx[j];
    }
    __syncthreads();
    float hr[RS_HPW][12];
#pragma unroll
    for (int k = 0; k < RS_HPW; ++k)
#pragma unroll
        for (int e = 0; e < 12; ++e) hr[k][e] = hs[warp * RS_HPW + k][e];
    int cnt[RS_HPW];
    double sum[RS_HPW];
#pragma unroll
    for (int k = 0; k < RS_HPW; ++k) { cnt[k] = 0; sum[k] = 0.0; }

    for (int base = 0; live && base < n; base += RS_TILE) {
        const int m = min(RS_TILE, n - base);
        __syncthreads();
        for (int e = threadIdx.x; e < 3 * m; e += blockDim.x) {
            tile[e % 3][e / 3] = src[3ll * base + e];
            tile[3 + e % 3][e / 3] = ref[3ll * base + e];
        }
        __syncthreads();
        for (int e = lane; e < m; e += 32) {
            const float x = tile[0][e], y = tile[1][e], z = tile[2][e], u = tile[3][e], v = tile[4][e], w = tile[5][e];
#pragma unroll
            for (int k = 0; k < RS_HPW; ++k) {
                const float d2 = rs_residual2(hr[k], x, y, z, u, v, w);
                if (d2 < tau2) { ++cnt[k]; sum[k] += (double)d2; }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < RS_HPW; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt[k] += __shfl_xor_sync(0xffffffffu, cnt[k], o);
        sum[k] = warp_sum_d(sum[k]);
    }
    if (lane < RS_HPW && h0 + lane < I) {
        int c = 0;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < RS_HPW; ++k) if (k == lane) { c = cnt[k]; s = sum[k]; }
        const float rmse = c > 0 ? (float)sqrt(s / (double)c) : 0.f;
        const long long q = (long long)p * I + h0 + lane;
        const float* o = hs[warp * RS_HPW + lane];
        for (int e = 0; e < 12; ++e) hyp_rt[12 * q + e] = o[e];
        hyp_cnt[q] = c;
        hyp_rmse[q] = rmse;
        if (rec_T != nullptr) {
            for (int e = 0; e < 12; ++e) rec_T[16 * q + e] = o[e];
            rec_T[16 * q + 12] = 0.f; rec_T[16 * q + 13] = 0.f; rec_T[16 * q + 14] = 0.f; rec_T[16 * q + 15] = 1.f;
        }
        if (rec_cnt != nullptr) rec_cnt[q] = c;
        if (rec_rmse != nullptr) rec_rmse[q] = rmse;
    }
}

// a better than b: more inliers, then lower rmse, then lower iteration (a strict total order: the reduction order is irrelevant)
__device__ __forceinline__ bool rs_better(int ca, float ra, int ia, int cb, float rb, int ib) {
    return ca > cb || (ca == cb && (ra < rb || (ra == rb && ia < ib)));
}

// Winner per pair: one CTA per pair (blockIdx.x), 256 threads.
__global__ void __launch_bounds__(256) ransac_select_kernel(const int* __restrict__ counts, int cap, int rn, int I,
                                                            const float* __restrict__ hyp_rt, const int* __restrict__ hyp_cnt,
                                                            const float* __restrict__ hyp_rmse, float* __restrict__ T,
                                                            float* __restrict__ fitness, float* __restrict__ rmse_out,
                                                            int* __restrict__ inliers, int* __restrict__ best_iter) {
    __shared__ int sc[256], si[256];
    __shared__ float sr[256];
    const int p = blockIdx.x, tid = threadIdx.x;
    const int n = rs_count(counts, p, cap);
    hyp_rt += 12ll * p * I; hyp_cnt += (long long)p * I; hyp_rmse += (long long)p * I;
    int bc = -1, bi = 0x7fffffff;
    float br = INFINITY;
    if (n >= rn)
        for (int i = tid; i < I; i += blockDim.x) {
            const int c = hyp_cnt[i];
            const float r = hyp_rmse[i];
            if (rs_better(c, r, i, bc, br, bi)) { bc = c; br = r; bi = i; }
        }
    sc[tid] = bc; sr[tid] = br; si[tid] = bi;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (tid < s && rs_better(sc[tid + s], sr[tid + s], si[tid + s], sc[tid], sr[tid], si[tid])) {
            sc[tid] = sc[tid + s]; sr[tid] = sr[tid + s]; si[tid] = si[tid + s];
        }
        __syncthreads();
    }
    const bool found = sc[0] > 0;            // a hypothesis without inliers never beats Open3D's default result
    if (tid < 16) {
        float v = (tid % 5 == 0) ? 1.f : 0.f;
        if (found && tid < 12) v = hyp_rt[12ll * si[0] + tid];
        T[16ll * p + tid] = v;
    }
    if (tid == 0) {
        fitness[p] = found ? (float)((double)sc[0] / (double)n) : 0.f;
        rmse_out[p] = found ? sr[0] : 0.f;
        inliers[p] = found ? sc[0] : 0;
        best_iter[p] = found ? si[0] : -1;
    }
}

// ---- correspondence metrics (evaluate_correspondences) ---------------------------------------------------------------------
// Grid (ceil(cap / 256), B): thread i of pair p takes correspondence i: its residual under T (inlier ratio, mean residual) and
// the distance from ref point i to the nearest transformed src correspondence point (overlap), brute force over smem tiles.
// Per-CTA partials [ir, ov, rs] go to part[p][blockIdx.x]; cm_finish_kernel sums them in order.
__global__ void __launch_bounds__(CM_THREADS) corr_metrics_kernel(const float* __restrict__ ref, const float* __restrict__ src, int cap,
                                                                  const int* __restrict__ counts, const float* __restrict__ T, int t_ld,
                                                                  float radius, double* __restrict__ part) {
    __shared__ float tile[3][CM_TILE];
    __shared__ float t[12];
    __shared__ double red[CM_THREADS / 32][3];
    const int p = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = rs_count(counts, p, cap);
    part += 3ll * ((long long)p * gridDim.x + blockIdx.x);
    if (blockIdx.x * CM_THREADS >= n) {
        if (threadIdx.x < 3) part[threadIdx.x] = 0.0;
        return;
    }
    ref += 3ll * p * cap; src += 3ll * p * cap;
    if (threadIdx.x < 12) t[threadIdx.x] = T[(long long)p * t_ld + threadIdx.x];
    __syncthreads();
    const int i = blockIdx.x * CM_THREADS + threadIdx.x;
    const bool act = i < n;
    float qx = 0.f, qy = 0.f, qz = 0.f, res = 0.f;
    if (act) {
        qx = ref[3 * i]; qy = ref[3 * i + 1]; qz = ref[3 * i + 2];
        const float x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
        const float ax = fmaf(z, t[2], fmaf(y, t[1], x * t[0])) + t[3];
        const float ay = fmaf(z, t[6], fmaf(y, t[5], x * t[4])) + t[7];
        const float az = fmaf(z, t[10], fmaf(y, t[9], x * t[8])) + t[11];
        const float dx = qx - ax, dy = qy - ay, dz = qz - az;
        res = sqrtf(dx * dx + dy * dy + dz * dz);
    }
    float best = INFINITY;
    for (int base = 0; base < n; base += CM_TILE) {
        const int m = min(CM_TILE, n - base);
        __syncthreads();
        for (int e = threadIdx.x; e < m; e += blockDim.x) {
            const float* s = src + 3ll * (base + e);
            const float x = s[0], y = s[1], z = s[2];
            tile[0][e] = fmaf(z, t[2], fmaf(y, t[1], x * t[0])) + t[3];
            tile[1][e] = fmaf(z, t[6], fmaf(y, t[5], x * t[4])) + t[7];
            tile[2][e] = fmaf(z, t[10], fmaf(y, t[9], x * t[8])) + t[11];
        }
        __syncthreads();
        if (act)
            for (int e = 0; e < m; ++e) {
                const float dx = qx - tile[0][e], dy = qy - tile[1][e], dz = qz - tile[2][e];
                best = fminf(best, dx * dx + dy * dy + dz * dz);
            }
    }
    double v[3] = {act && res < radius ? 1.0 : 0.0, act && sqrtf(best) < radius ? 1.0 : 0.0, act ? (double)res : 0.0};
    for (int k = 0; k < 3; ++k) v[k] = warp_sum_d(v[k]);
    if (lane == 0) for (int k = 0; k < 3; ++k) red[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x < 3) {
        double s = 0.0;
        for (int w = 0; w < CM_THREADS / 32; ++w) s += red[w][threadIdx.x];
        part[threadIdx.x] = s;
    }
}

// one warp per pair: [f_IR, f_OV, f_RS, f_NU]; the means of an empty set are NaN (numpy's mean of an empty array)
__global__ void __launch_bounds__(32) cm_finish_kernel(const double* __restrict__ part, int nblk, const int* __restrict__ counts, int cap,
                                                       float* __restrict__ out, int out_ld) {
    const int p = blockIdx.x, lane = threadIdx.x;
    const int n = rs_count(counts, p, cap);
    part += 3ll * p * nblk;
    double v[3] = {0.0, 0.0, 0.0};
    for (int b = lane; b < nblk; b += 32)
        for (int k = 0; k < 3; ++k) v[k] += part[3 * b + k];
    for (int k = 0; k < 3; ++k) v[k] = warp_sum_d(v[k]);
    if (lane == 0) {
        float* o = out + (long long)p * out_ld;
        const double inv = n > 0 ? 1.0 / (double)n : __longlong_as_double(0x7ff8000000000000ll);
        o[0] = (float)(v[0] * inv); o[1] = (float)(v[1] * inv); o[2] = (float)(v[2] * inv); o[3] = (float)n;
    }
}

// ---- feature-matching RANSAC (utils/open3d.py:133-166, Open3D 0.11 registration_ransac_based_on_feature_matching) ---------------
// The src -> ref descriptor matches come from feature_match.cu.  Then, per pair (DESIGN.md section 3b):
//   build     one thread per iteration: Philox sample (the stream above), edge-length check, Kabsch, distance check -> pass flag;
//   validate  one CTA per pair: ordered prefix count over the pass flags -> the first V passing iterations;
//   grid      a hashed uniform grid of the ref cloud (cell 1.001 tau, so every point within tau lies in the 27 cells around);
//   score     one CTA per validated hypothesis: every src point transformed (pinned fp32), nearest ref point over the 27 cells;
//   select    ransac_select_kernel over the validated slots (slot order = iteration order), then slot -> iteration.
constexpr int FR_THREADS = 128, FR_SCORE_THREADS = 256;
constexpr double FR_CELL = 1.001;

// Grid (ceil(I / 128), B).  Iteration i of pair p; coordinates in double, every operation rounded on its own.
__global__ void __launch_bounds__(FR_THREADS) fr_build_kernel(const float* __restrict__ src, const float* __restrict__ ref, int cap_s, int cap_r,
                                                              const int32_t* __restrict__ ns_c, const int32_t* __restrict__ nr_c,
                                                              const int64_t* __restrict__ match, double tau, int rn, int I, uint32_t key0,
                                                              uint32_t key1, uint32_t pair_base, float* __restrict__ hyp_rt,
                                                              int* __restrict__ pass, int* __restrict__ rec_samples) {
    const int p = blockIdx.y, i = blockIdx.x * FR_THREADS + threadIdx.x;
    if (i >= I) return;
    const int n = rs_count(ns_c, p, cap_s), nr = rs_count(nr_c, p, cap_r);
    src += 3ll * p * cap_s; ref += 3ll * p * cap_r; match += (long long)p * cap_s;
    int idx[RS_MAX_N];
#pragma unroll
    for (int j = 0; j < RS_MAX_N; ++j) idx[j] = -1;
    int ok = 0;
    if (n >= rn && nr > 0) {
        uint32_t c[4];
        float s[RS_MAX_N][3], t[RS_MAX_N][3];
#pragma unroll
        for (int j = 0; j < RS_MAX_N; ++j) {
            if (j % 4 == 0) { c[0] = (uint32_t)i; c[1] = pair_base + (uint32_t)p; c[2] = (uint32_t)(j / 4); c[3] = 0u; philox4x32_10(c, key0, key1); }
            if (j < rn) {
                idx[j] = (int)__umulhi(c[j % 4], (uint32_t)n);
                const long long m = match[idx[j]];
                for (int a = 0; a < 3; ++a) { s[j][a] = src[3 * idx[j] + a]; t[j][a] = ref[3 * m + a]; }
            }
        }
        ok = 1;
        // CorrespondenceCheckerBasedOnEdgeLength(0.9): every edge of the sample, |s_j - s_k| against |t_j - t_k|
#pragma unroll
        for (int j = 0; j < RS_MAX_N; ++j)
#pragma unroll
            for (int k = j + 1; k < RS_MAX_N; ++k)
                if (k < rn) {
                    double ds = 0.0, dt = 0.0;
                    for (int a = 0; a < 3; ++a) {
                        const double u = __dsub_rn((double)s[j][a], (double)s[k][a]), v = __dsub_rn((double)t[j][a], (double)t[k][a]);
                        ds = __dadd_rn(ds, __dmul_rn(u, u)); dt = __dadd_rn(dt, __dmul_rn(v, v));
                    }
                    ds = sqrt(ds); dt = sqrt(dt);
                    if (ds < __dmul_rn(0.9, dt) || dt < __dmul_rn(0.9, ds)) ok = 0;
                }
        if (ok) {
            double cs[3] = {0, 0, 0}, cr[3] = {0, 0, 0};
#pragma unroll
            for (int j = 0; j < RS_MAX_N; ++j)
                if (j < rn)
                    for (int a = 0; a < 3; ++a) { cs[a] += (double)s[j][a]; cr[a] += (double)t[j][a]; }
            for (int a = 0; a < 3; ++a) { cs[a] /= rn; cr[a] /= rn; }
            double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, R[9], tr[3];
#pragma unroll
            for (int j = 0; j < RS_MAX_N; ++j)
                if (j < rn)
                    for (int a = 0; a < 3; ++a)
                        for (int b = 0; b < 3; ++b) H[3 * a + b] += ((double)s[j][a] - cs[a]) * ((double)t[j][b] - cr[b]);
            kabsch_rotation(H, R);
            for (int a = 0; a < 3; ++a) tr[a] = cr[a] - (R[3 * a] * cs[0] + R[3 * a + 1] * cs[1] + R[3 * a + 2] * cs[2]);
            // CorrespondenceCheckerBasedOnDistance(tau): |R s_j + t - t_j| <= tau for every sample, on the double (R, t)
#pragma unroll
            for (int j = 0; j < RS_MAX_N; ++j)
                if (j < rn) {
                    double d2 = 0.0;
                    for (int a = 0; a < 3; ++a) {
                        const double y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[3 * a], (double)s[j][0]), __dmul_rn(R[3 * a + 1], (double)s[j][1])),
                                                             __dmul_rn(R[3 * a + 2], (double)s[j][2])), tr[a]);
                        const double e = __dsub_rn(y, (double)t[j][a]);
                        d2 = __dadd_rn(d2, __dmul_rn(e, e));
                    }
                    if (sqrt(d2) > tau) ok = 0;
                }
            if (ok) {
                float* o = hyp_rt + 12 * ((long long)p * I + i);
                for (int a = 0; a < 3; ++a) {
                    for (int b = 0; b < 3; ++b) o[4 * a + b] = (float)R[3 * a + b];
                    o[4 * a + 3] = (float)tr[a];
                }
            }
        }
    }
    pass[(long long)p * I + i] = ok;
    if (rec_samples != nullptr)
        for (int j = 0; j < RS_MAX_N; ++j) rec_samples[((long long)p * I + i) * RS_MAX_N + j] = idx[j];
}

// One CTA of 1024 threads per pair: val_ids[p][k] = the k-th passing iteration (k < V), -1 beyond; nval[p] = their number.
__global__ void __launch_bounds__(1024) fr_validate_kernel(const int* __restrict__ pass, int I, int V, int* __restrict__ val_ids,
                                                           int32_t* __restrict__ nval) {
    __shared__ int wsum[32];
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pass += (long long)p * I; val_ids += (long long)p * V;
    int base = 0;
    for (int c0 = 0; c0 < I && base < V; c0 += 1024) {              // base is uniform over the CTA
        const int i = c0 + tid;
        const int f = i < I ? pass[i] : 0;
        int incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int w = wsum[lane];
            int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += v;
            }
            wsum[lane] = wi - w;
        }
        __syncthreads();
        const int k = base + wsum[warp] + incl - f;
        if (f && k < V) val_ids[k] = i;
        const int last = __shfl_sync(0xffffffffu, wsum[warp] + incl, 31);
        __syncthreads();
        if (tid == 1023) wsum[0] = last;
        __syncthreads();
        base += wsum[0];
        __syncthreads();
    }
    const int nv = min(base, V);
    for (int k = nv + tid; k < V; k += 1024) val_ids[k] = -1;
    if (tid == 0) nval[p] = nv;
}

__device__ __forceinline__ long long fr_cell(float x, double inv_cell) {
    return (long long)fmin(fmax(floor((double)x * inv_cell), -1e15), 1e15);
}

__device__ __forceinline__ int fr_hash(long long x, long long y, long long z, int H) {
    return (int)(((unsigned long long)x * 73856093ull ^ (unsigned long long)y * 19349663ull ^ (unsigned long long)z * 83492791ull) &
                 (unsigned long long)(H - 1));
}

// Grid (ceil(cap_r / 256), B): bucket of every ref point, and the bucket sizes.
__global__ void __launch_bounds__(256) fr_hash_kernel(const float* __restrict__ ref, int cap_r, const int32_t* __restrict__ nr_c, double inv_cell,
                                                      int H, int* __restrict__ key, int* __restrict__ bcount) {
    const int p = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
    if (j >= rs_count(nr_c, p, cap_r)) return;
    const float* r = ref + 3ll * ((long long)p * cap_r + j);
    const int b = fr_hash(fr_cell(r[0], inv_cell), fr_cell(r[1], inv_cell), fr_cell(r[2], inv_cell), H);
    key[(long long)p * cap_r + j] = b;
    atomicAdd(bcount + (long long)p * (H + 1) + b, 1);
}

// One CTA of 1024 threads per pair: bucket sizes -> exclusive bucket starts (entry H = the point count), copied to the cursors.
__global__ void __launch_bounds__(1024) fr_scan_kernel(int* __restrict__ bstart, int* __restrict__ cursor, int H) {
    __shared__ int wsum[32];
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    bstart += (long long)p * (H + 1); cursor += (long long)p * (H + 1);
    int base = 0;
    for (int c0 = 0; c0 <= H; c0 += 1024) {
        const int i = c0 + tid;
        const int f = i < H ? bstart[i] : 0;
        int incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int w = wsum[lane];
            int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += v;
            }
            wsum[lane] = wi - w;
        }
        __syncthreads();
        const int start = base + wsum[warp] + incl - f;
        if (i <= H) { bstart[i] = start; cursor[i] = start; }
        const int last = __shfl_sync(0xffffffffu, wsum[warp] + incl, 31);
        __syncthreads();
        if (tid == 1023) wsum[0] = last;
        __syncthreads();
        base += wsum[0];
        __syncthreads();
    }
}

// Ref points into bucket order (the order inside a bucket is arbitrary: the score only takes minima over it).
__global__ void __launch_bounds__(256) fr_scatter_kernel(const float* __restrict__ ref, int cap_r, const int32_t* __restrict__ nr_c, int H,
                                                         const int* __restrict__ key, int* __restrict__ cursor, float4* __restrict__ sorted) {
    const int p = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
    if (j >= rs_count(nr_c, p, cap_r)) return;
    const long long q = (long long)p * cap_r + j;
    const int pos = atomicAdd(cursor + (long long)p * (H + 1) + key[q], 1);
    sorted[(long long)p * cap_r + pos] = make_float4(ref[3 * q], ref[3 * q + 1], ref[3 * q + 2], 0.f);
}

// Grid (V, B), 256 threads: validated slot v of pair p.  Per src point: position under (R, t) as rs_residual2 forms it, nearest
// ref point over the 27 cells with d^2 = (dx^2 + dy^2) + dz^2 pinned; inlier when d^2 < tau^2.  Fixed reduction order.
__global__ void __launch_bounds__(FR_SCORE_THREADS, 1) fr_score_kernel(const float* __restrict__ src, int cap_s, int cap_r,
                                                                    const int32_t* __restrict__ ns_c, const float* __restrict__ hyp_rt, int I,
                                                                    const int* __restrict__ val_ids, const int32_t* __restrict__ nval, int V,
                                                                    const int* __restrict__ bstart, const float4* __restrict__ sorted, int H,
                                                                    double inv_cell, float tau2, float* __restrict__ v_rt,
                                                                    int* __restrict__ v_cnt, float* __restrict__ v_rmse,
                                                                    float* __restrict__ rec_T) {
    __shared__ float h[12];
    __shared__ int rc[FR_SCORE_THREADS / 32];
    __shared__ double rsum[FR_SCORE_THREADS / 32];
    const int p = blockIdx.y, v = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long q = (long long)p * V + v;
    const bool live = v < nval[p];
    if (tid < 12) h[tid] = live ? hyp_rt[12 * ((long long)p * I + val_ids[q]) + tid] : ((tid % 5 == 0) ? 1.f : 0.f);
    __syncthreads();
    int cnt = 0;
    double sum = 0.0;
    if (live) {
        const int n = rs_count(ns_c, p, cap_s);
        src += 3ll * p * cap_s; bstart += (long long)p * (H + 1); sorted += (long long)p * cap_r;
        for (int j = tid; j < n; j += FR_SCORE_THREADS) {
            const float x = src[3 * j], y = src[3 * j + 1], z = src[3 * j + 2];
            const float ax = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(h[0], x), __fmul_rn(h[1], y)), __fmul_rn(h[2], z)), h[3]);
            const float ay = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(h[4], x), __fmul_rn(h[5], y)), __fmul_rn(h[6], z)), h[7]);
            const float az = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(h[8], x), __fmul_rn(h[9], y)), __fmul_rn(h[10], z)), h[11]);
            const long long cx = fr_cell(ax, inv_cell), cy = fr_cell(ay, inv_cell), cz = fr_cell(az, inv_cell);
            float best = INFINITY;
#pragma unroll 1
            for (int cell = 0; cell < 27; ++cell) {
                const int b = fr_hash(cx + cell % 3 - 1, cy + (cell / 3) % 3 - 1, cz + cell / 9 - 1, H);
                const int e = bstart[b + 1];
                for (int k = bstart[b]; k < e; ++k) {
                    const float4 r = sorted[k];
                    const float ex = __fsub_rn(ax, r.x), ey = __fsub_rn(ay, r.y), ez = __fsub_rn(az, r.z);
                    best = fminf(best, __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)));
                }
            }
            if (best < tau2) { ++cnt; sum += (double)best; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    sum = warp_sum_d(sum);
    if (lane == 0) { rc[warp] = cnt; rsum[warp] = sum; }
    __syncthreads();
    if (tid < 12) v_rt[12 * q + tid] = h[tid];
    if (rec_T != nullptr && tid < 16) rec_T[16 * q + tid] = tid < 12 ? h[tid] : (tid == 15 ? 1.f : 0.f);
    if (tid == 0) {
        int c = 0;
        double s = 0.0;
        for (int w = 0; w < FR_SCORE_THREADS / 32; ++w) { c += rc[w]; s += rsum[w]; }
        v_cnt[q] = c;
        v_rmse[q] = c > 0 ? (float)__dsqrt_rn(__ddiv_rn(s, (double)c)) : 0.f;
    }
}

// slot -> iteration; the default result for the degenerate arguments (no launch of the pipeline at all)
__global__ void fr_finish_kernel(int B, const int* __restrict__ val_ids, int V, int* __restrict__ best_iter, float* __restrict__ T,
                                 float* __restrict__ fitness, float* __restrict__ rmse, int* __restrict__ inliers, int32_t* __restrict__ nval,
                                 bool degenerate) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= B) return;
    if (degenerate) {
        for (int e = 0; e < 16; ++e) T[16ll * p + e] = (e % 5 == 0) ? 1.f : 0.f;
        fitness[p] = 0.f; rmse[p] = 0.f; inliers[p] = 0; best_iter[p] = -1; nval[p] = 0;
    } else if (best_iter[p] >= 0) {
        best_iter[p] = val_ids[(long long)p * V + best_iter[p]];
    }
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_ransac_correspondences_batched_workspace_bytes(int64_t n_pairs, int64_t num_iterations) {
    const size_t h = (size_t)(n_pairs > 0 ? n_pairs : 0) * (size_t)(num_iterations > 0 ? num_iterations : 0);
    return align_up(12 * 4 * h, 256) + 2 * align_up(4 * h, 256) + 256;
}

int geob200_ransac_correspondences_batched(const float* ref_corr_points, const float* src_corr_points, int64_t n_pairs, int64_t capacity,
                                           const int32_t* num_corr, float distance_threshold, int64_t ransac_n, int64_t num_iterations,
                                           uint64_t seed, int64_t pair_base, float* transforms, float* fitness, float* inlier_rmse, int32_t* inlier_count,
                                           int32_t* best_iteration, float* hyp_transforms, int32_t* hyp_inliers, float* hyp_rmse,
                                           int32_t* hyp_samples, void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(ransac_n >= 3 && ransac_n <= RS_MAX_N, "ransac: ransac_n must be in 3..%d", RS_MAX_N);
    GEOB_REQUIRE(num_iterations > 0 && num_iterations <= (1ll << 30), "ransac: num_iterations must be in 1..2^30");
    GEOB_REQUIRE(distance_threshold > 0.f, "ransac: distance_threshold must be > 0");
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "ransac: 1..65535 pairs");
    GEOB_REQUIRE(pair_base >= 0 && pair_base + n_pairs <= (1ll << 32), "ransac: pair ids must fit 32 bits");
    GEOB_REQUIRE(capacity >= 0 && capacity < (1ll << 31) / 3, "ransac: bad capacity");
    GEOB_REQUIRE((ref_corr_points != nullptr && src_corr_points != nullptr) || capacity == 0, "ransac: null correspondence points");
    GEOB_REQUIRE(transforms != nullptr && fitness != nullptr && inlier_rmse != nullptr && inlier_count != nullptr &&
                     best_iteration != nullptr, "ransac: null output");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_ransac_correspondences_batched_workspace_bytes(n_pairs, num_iterations),
                 "ransac: workspace too small");
    Arena ar(workspace, workspace_bytes);
    const size_t h = (size_t)n_pairs * (size_t)num_iterations;
    float* hyp_rt = ar.take<float>(12 * h);
    int* hcnt = ar.take<int>(h);
    float* hrmse = ar.take<float>(h);
    GEOB_REQUIRE(ar.ok(), "ransac: workspace too small");
    const int I = (int)num_iterations, B = (int)n_pairs, cap = (int)capacity, rn = (int)ransac_n;
    const float tau2 = distance_threshold * distance_threshold;
    cudaStream_t st = (cudaStream_t)stream;
    ransac_hypotheses_kernel<<<dim3((unsigned)((I + RS_HPB - 1) / RS_HPB), B), RS_WARPS * 32, 0, st>>>(
        ref_corr_points, src_corr_points, cap, num_corr, tau2, rn, I, (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)pair_base, hyp_rt, hcnt, hrmse,
        hyp_transforms, hyp_inliers, hyp_rmse, hyp_samples);
    ransac_select_kernel<<<B, 256, 0, st>>>(num_corr, cap, rn, I, hyp_rt, hcnt, hrmse, transforms, fitness, inlier_rmse, inlier_count,
                                            best_iteration);
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

static int fr_hash_size(int64_t cap_ref) {
    int H = 1024;
    while (H < 2 * cap_ref) H <<= 1;
    return H;
}

size_t geob200_ransac_features_batched_workspace_bytes(int64_t n_pairs, int64_t cap_src, int64_t cap_ref, int64_t num_iterations,
                                                       int64_t val_iterations) {
    const size_t B = (size_t)(n_pairs > 0 ? n_pairs : 0), cs = (size_t)(cap_src > 0 ? cap_src : 0), cr = (size_t)(cap_ref > 0 ? cap_ref : 0);
    const size_t I = (size_t)(num_iterations > 0 ? num_iterations : 0);
    const size_t V = std::min(I, (size_t)(val_iterations > 0 ? val_iterations : 0));
    const size_t H = (size_t)fr_hash_size((int64_t)cr);
    return feature_nn_workspace(n_pairs, cap_src, cap_ref) + align_up(8 * B * cs, 256) + align_up(8 * B * cs, 256) +
           align_up(48 * B * I, 256) + align_up(4 * B * I, 256) + align_up(4 * B * V, 256) + align_up(48 * B * V, 256) +
           2 * align_up(4 * B * V, 256) + 2 * align_up(4 * B * (H + 1), 256) + align_up(4 * B * cr, 256) + align_up(16 * B * cr, 256) + 256;
}

int geob200_ransac_features_batched(const float* src_points, const float* ref_points, const float* src_feats, const float* ref_feats,
                                    int64_t n_pairs, int64_t cap_src, int64_t cap_ref, int64_t channels, const int32_t* n_src,
                                    const int32_t* n_ref, float distance_threshold, int64_t ransac_n, int64_t num_iterations,
                                    int64_t val_iterations, uint64_t seed, int64_t pair_base, float* transforms, float* fitness,
                                    float* inlier_rmse, int32_t* inlier_count, int32_t* best_iteration, int32_t* num_validated,
                                    int64_t* rec_matches, int32_t* rec_samples, int32_t* rec_pass, int32_t* rec_val_ids,
                                    float* rec_transforms, int32_t* rec_inliers, float* rec_rmse, void* workspace, size_t workspace_bytes,
                                    void* stream) {
    GEOB_REQUIRE(ransac_n >= 0 && ransac_n <= RS_MAX_N, "ransac_features: ransac_n must be in 0..%d", RS_MAX_N);
    GEOB_REQUIRE(num_iterations >= 0 && num_iterations <= (1ll << 30), "ransac_features: num_iterations must be in 0..2^30");
    GEOB_REQUIRE(val_iterations >= 0 && val_iterations <= (1ll << 30), "ransac_features: val_iterations must be in 0..2^30");
    GEOB_REQUIRE(channels >= 1 && channels <= 1024, "ransac_features: channels must be in 1..1024");
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "ransac_features: 1..65535 pairs");
    GEOB_REQUIRE(pair_base >= 0 && pair_base + n_pairs <= (1ll << 32), "ransac_features: pair ids must fit 32 bits");
    GEOB_REQUIRE(cap_src >= 0 && cap_ref >= 0 && cap_src < (1ll << 28) && cap_ref < (1ll << 28), "ransac_features: capacities must be in 0..2^28");
    GEOB_REQUIRE((src_points != nullptr && src_feats != nullptr) || cap_src == 0, "ransac_features: null src points / descriptors");
    GEOB_REQUIRE((ref_points != nullptr && ref_feats != nullptr) || cap_ref == 0, "ransac_features: null ref points / descriptors");
    GEOB_REQUIRE(transforms != nullptr && fitness != nullptr && inlier_rmse != nullptr && inlier_count != nullptr && best_iteration != nullptr &&
                     num_validated != nullptr, "ransac_features: null output");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_ransac_features_batched_workspace_bytes(n_pairs, cap_src, cap_ref,
                                                                                                          num_iterations, val_iterations),
                 "ransac_features: workspace too small");
    const int B = (int)n_pairs, cs = (int)cap_src, cr = (int)cap_ref, rn = (int)ransac_n, I = (int)num_iterations;
    const int V = (int)std::min(num_iterations, val_iterations), H = fr_hash_size(cap_ref);
    cudaStream_t st = (cudaStream_t)stream;
    if (rn < 3 || !(distance_threshold > 0.f) || V == 0) {      // Open3D's default result
        fr_finish_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, nullptr, 0, best_iteration, transforms, fitness, inlier_rmse, inlier_count,
                                                          num_validated, true);
        GEOB_CHECK_LAUNCH();
        count_launches(1);
        return 0;
    }
    const size_t nn_ws = feature_nn_workspace(n_pairs, cap_src, cap_ref);
    Arena ar((char*)workspace + nn_ws, workspace_bytes - nn_ws);
    int64_t* match = ar.take<int64_t>((size_t)B * cs);
    double* mdist = ar.take<double>((size_t)B * cs);
    float* hyp_rt = ar.take<float>((size_t)B * I * 12);
    int* pass = ar.take<int>((size_t)B * I);
    int* val_ids = ar.take<int>((size_t)B * V);
    float* v_rt = ar.take<float>((size_t)B * V * 12);
    int* v_cnt = ar.take<int>((size_t)B * V);
    float* v_rmse = ar.take<float>((size_t)B * V);
    int* bstart = ar.take<int>((size_t)B * (H + 1));
    int* cursor = ar.take<int>((size_t)B * (H + 1));
    int* key = ar.take<int>((size_t)B * cr);
    float4* sorted = ar.take<float4>((size_t)B * cr);
    GEOB_REQUIRE(ar.ok(), "ransac_features: workspace too small");
    if (rec_matches != nullptr) match = rec_matches;
    if (rec_pass != nullptr) pass = rec_pass;
    if (rec_val_ids != nullptr) val_ids = rec_val_ids;
    if (rec_inliers != nullptr) v_cnt = rec_inliers;
    if (rec_rmse != nullptr) v_rmse = rec_rmse;
    int nl = 0;
    if (feature_nn_launch(src_feats, ref_feats, B, cs, cr, (int)channels, n_src, n_ref, match, mdist, nullptr, nullptr, workspace, nn_ws, st,
                          &nl) != 0)
        return -1;
    const double tau = (double)distance_threshold, inv_cell = 1.0 / (FR_CELL * tau);
    fr_build_kernel<<<dim3((unsigned)((I + FR_THREADS - 1) / FR_THREADS), B), FR_THREADS, 0, st>>>(
        src_points, ref_points, cs, cr, n_src, n_ref, match, tau, rn, I, (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)pair_base, hyp_rt,
        pass, rec_samples);
    fr_validate_kernel<<<B, 1024, 0, st>>>(pass, I, V, val_ids, num_validated);
    GEOB_CHECK_CUDA(cudaMemsetAsync(bstart, 0, 4 * (size_t)B * (H + 1), st));
    nl += 2;
    if (cr > 0) {
        fr_hash_kernel<<<dim3((cr + 255) / 256, B), 256, 0, st>>>(ref_points, cr, n_ref, inv_cell, H, key, bstart);
        fr_scan_kernel<<<B, 1024, 0, st>>>(bstart, cursor, H);
        fr_scatter_kernel<<<dim3((cr + 255) / 256, B), 256, 0, st>>>(ref_points, cr, n_ref, H, key, cursor, sorted);
        nl += 3;
    }
    fr_score_kernel<<<dim3((unsigned)V, B), FR_SCORE_THREADS, 0, st>>>(src_points, cs, cr, n_src, hyp_rt, I, val_ids, num_validated, V, bstart,
                                                                       sorted, H, inv_cell, (float)(distance_threshold * distance_threshold),
                                                                       v_rt, v_cnt, v_rmse, rec_transforms);
    ransac_select_kernel<<<B, 256, 0, st>>>(n_src, cs, rn, V, v_rt, v_cnt, v_rmse, transforms, fitness, inlier_rmse, inlier_count,
                                            best_iteration);
    fr_finish_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, val_ids, V, best_iteration, transforms, fitness, inlier_rmse, inlier_count,
                                                      num_validated, false);
    nl += 3;
    GEOB_CHECK_LAUNCH();
    count_launches(nl);
    return 0;
}

size_t geob200_correspondence_metrics_batched_workspace_bytes(int64_t n_pairs, int64_t capacity) {
    const size_t nblk = (size_t)((capacity > 0 ? capacity : 0) + CM_THREADS - 1) / CM_THREADS;
    return align_up(3 * 8 * (size_t)(n_pairs > 0 ? n_pairs : 0) * (nblk > 0 ? nblk : 1), 256) + 256;
}

int geob200_correspondence_metrics_batched(const float* ref_corr_points, const float* src_corr_points, int64_t n_pairs, int64_t capacity,
                                           const int32_t* num_corr, const float* transforms, int64_t transform_ld, float positive_radius,
                                           float* out, int64_t out_ld, void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "correspondence_metrics: 1..65535 pairs");
    GEOB_REQUIRE(capacity >= 0 && capacity < (1ll << 31) / 3, "correspondence_metrics: bad capacity");
    GEOB_REQUIRE((ref_corr_points != nullptr && src_corr_points != nullptr) || capacity == 0, "correspondence_metrics: null points");
    GEOB_REQUIRE(transforms != nullptr && transform_ld >= 12 && out != nullptr && out_ld >= 4, "correspondence_metrics: bad output");
    GEOB_REQUIRE(positive_radius > 0.f, "correspondence_metrics: positive_radius must be > 0");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_correspondence_metrics_batched_workspace_bytes(n_pairs, capacity),
                 "correspondence_metrics: workspace too small");
    const int nblk = (int)((capacity + CM_THREADS - 1) / CM_THREADS);
    double* part = (double*)workspace;
    cudaStream_t st = (cudaStream_t)stream;
    if (nblk > 0)
        corr_metrics_kernel<<<dim3(nblk, (unsigned)n_pairs), CM_THREADS, 0, st>>>(ref_corr_points, src_corr_points, (int)capacity, num_corr,
                                                                                  transforms, (int)transform_ld, positive_radius, part);
    cm_finish_kernel<<<(unsigned)n_pairs, 32, 0, st>>>(part, nblk, num_corr, (int)capacity, out, (int)out_ld);
    GEOB_CHECK_LAUNCH();
    count_launches(nblk > 0 ? 2 : 1);
    return 0;
}

}  // extern "C"
