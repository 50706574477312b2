// Local-to-Global Registration: dense correspondences from the patch assignment matrices, per-patch weighted
// Kabsch hypotheses, hypothesis verification, iterative weighted-SVD refinement.
//
// Reference: geotransformer/modules/geotransformer/local_global_registration.py:49-235 and
//            geotransformer/modules/registration/procrustes.py:6-73 (torch.svd on the HOST, six D2H/H2D round trips per
//            pair, plus .tolist() and Python chunk lists).  Here everything stays on the device: no host round trip.
#include "common.cuh"
#include "geob200.h"
#include "kabsch.cuh"

namespace geob200 {

// transform (row-major 4x4 fp32) from accumulated moments: sw = sum w_raw ; the normalised weights are
// w_raw/(sw+eps) (procrustes.py:44).  S1 = sum w x (src), S2 = sum w y (ref), Sxy[a][b] = sum w x_a y_b, all with
// NORMALISED weights w and W = sum w.  H = sum w (x-cx)(y-cy)^T with cx = S1 (centroids use the same weights, which
// do not sum exactly to one) = Sxy - cx S2^T - S1 cy^T + W cx cy^T.
__device__ void finish_procrustes(double W, const double S1[3], const double S2[3], const double Sxy[9], float* T) {
    double H[9], R[9];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) H[3 * a + b] = Sxy[3 * a + b] - S1[a] * S2[b] - S1[a] * S2[b] + W * S1[a] * S2[b];
    kabsch_rotation(H, R);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[4 * i + j] = (float)R[3 * i + j];
        T[4 * i + 3] = (float)(S2[i] - (R[3 * i] * S1[0] + R[3 * i + 1] * S1[1] + R[3 * i + 2] * S1[2]));   // t = cy - R cx
    }
    T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
}

// ---- correspondence extraction ---------------------------------------------------------------------------
// One CTA per patch pair.  score = exp(log-assignment[:K,:K]); mutual top-k over rows and columns, > confidence,
// both points valid (local_global_registration.py:49-83).  Emits the patch's correspondences in (i,j) row-major order.
template <int TOPK_MAX>
__global__ void __launch_bounds__(256) lgr_corr_kernel(const float* __restrict__ log_scores, int K, int ld /*K or K+1*/,
                                                       const unsigned char* __restrict__ ref_masks, const unsigned char* __restrict__ src_masks,
                                                       int topk, float conf, int mutual, int* __restrict__ patch_count,
                                                       int* __restrict__ patch_ij /*[P][K*topk]*/, float* __restrict__ patch_score) {
    extern __shared__ float sm[];
    float* sc = sm;                                   // [K][K+1]
    unsigned char* rsel = (unsigned char*)(sc + K * (K + 1));   // [K][K]
    unsigned char* csel = rsel + K * K;
    __shared__ int row_cnt[256];
    const int p = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sld = K + 1;
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
        const int i = e / K, j = e % K;
        sc[i * sld + j] = expf(log_scores[((long long)p * ld + i) * ld + j]);
        rsel[e] = 0; csel[e] = 0;
    }
    __syncthreads();
    // row top-k (ties: lowest column), column top-k (ties: lowest row)
    for (int i = warp; i < K; i += 8) {
        int taken[TOPK_MAX];
        for (int r = 0; r < topk; ++r) {
            float bv = -INFINITY; int bj = 0x7fffffff;
            for (int j = lane; j < K; j += 32) {
                bool skip = false;
                for (int q = 0; q < r; ++q) skip |= (taken[q] == j);
                const float v = sc[i * sld + j];
                if (!skip && (v > bv || (v == bv && j < bj))) { bv = v; bj = j; }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
                if (ov > bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
            }
            taken[r] = bj;
            if (lane == 0 && bj < K && bv > conf) rsel[i * K + bj] = 1;
        }
    }
    for (int j = warp; j < K; j += 8) {
        int taken[TOPK_MAX];
        for (int r = 0; r < topk; ++r) {
            float bv = -INFINITY; int bi = 0x7fffffff;
            for (int i = lane; i < K; i += 32) {
                bool skip = false;
                for (int q = 0; q < r; ++q) skip |= (taken[q] == i);
                const float v = sc[i * sld + j];
                if (!skip && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            taken[r] = bi;
            if (lane == 0 && bi < K && bv > conf) csel[bi * K + j] = 1;
        }
    }
    __syncthreads();
    // final flags + ordered compaction (row-major)
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        int c = 0;
        const bool rm = ref_masks[(long long)p * K + i];
        for (int j = 0; j < K; ++j) {
            const bool f = (mutual ? (rsel[i * K + j] && csel[i * K + j]) : (rsel[i * K + j] || csel[i * K + j])) && rm &&
                           src_masks[(long long)p * K + j];
            rsel[i * K + j] = f ? 1 : 0;
            c += f ? 1 : 0;
        }
        row_cnt[i] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int i = 0; i < K; ++i) { const int c = row_cnt[i]; row_cnt[i] = acc; acc += c; }
        patch_count[p] = acc;
    }
    __syncthreads();
    const int cap = K * (mutual ? topk : 2 * topk);
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        int o = row_cnt[i];
        for (int j = 0; j < K; ++j)
            if (rsel[i * K + j]) {
                patch_ij[(long long)p * cap + o] = i * K + j;
                patch_score[(long long)p * cap + o] = sc[i * sld + j];
                ++o;
            }
    }
}

// offsets over the P patches of pair blockIdx.x (one CTA per pair), total count
__global__ void __launch_bounds__(1024) lgr_offsets_kernel(const int* __restrict__ patch_count, int P, int* __restrict__ patch_off,
                                                           int* __restrict__ total) {
    patch_count += (long long)blockIdx.x * P;
    patch_off += (long long)blockIdx.x * (P + 1);
    total += blockIdx.x;
    __shared__ int carry;
    __shared__ int warp_tot[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < P; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = (i < P) ? patch_count[i] : 0;
        int x = v;
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        if (lane == 31) warp_tot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int w = warp_tot[lane];
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
            warp_tot[lane] = w;
        }
        __syncthreads();
        if (i < P) patch_off[i] = carry + (warp > 0 ? warp_tot[warp - 1] : 0) + x - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += warp_tot[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) { patch_off[P] = carry; *total = carry; }
}

// stacked correspondences in (patch, i, j) order (local_global_registration.py:139-142).  Patch blockIdx.x of pair blockIdx.y
// (gridDim.x patches per pair); the pair's rows start at blockIdx.y * gridDim.x * cap.
__global__ void __launch_bounds__(256) lgr_stack_kernel(const int* __restrict__ patch_count, const int* __restrict__ patch_off,
                                                        const int* __restrict__ patch_ij, const float* __restrict__ patch_score, int K,
                                                        int cap, const float* __restrict__ ref_knn_pts, const float* __restrict__ src_knn_pts,
                                                        float* __restrict__ ref_corr, float* __restrict__ src_corr,
                                                        float* __restrict__ corr_scores, int* __restrict__ corr_patch) {
    const int P = gridDim.x, b = blockIdx.y;
    const long long first = (long long)b * P * cap;
    ref_corr += 3 * first; src_corr += 3 * first; corr_scores += first; corr_patch += first;
    const int c = patch_count[b * P + blockIdx.x], off = patch_off[b * (P + 1) + blockIdx.x];
    const long long p = (long long)b * P + blockIdx.x;
    for (int e = threadIdx.x; e < c; e += blockDim.x) {
        const int ij = patch_ij[(long long)p * cap + e];
        const int i = ij / K, j = ij % K;
        const float* r = ref_knn_pts + ((long long)p * K + i) * 3;
        const float* s = src_knn_pts + ((long long)p * K + j) * 3;
        const long long o = off + e;
        ref_corr[3 * o] = r[0]; ref_corr[3 * o + 1] = r[1]; ref_corr[3 * o + 2] = r[2];
        src_corr[3 * o] = s[0]; src_corr[3 * o + 1] = s[1]; src_corr[3 * o + 2] = s[2];
        corr_scores[o] = patch_score[(long long)p * cap + e];
        corr_patch[o] = blockIdx.x;
    }
}

// per-patch weighted Kabsch (one warp per patch); patches with < min_corr correspondences are marked invalid.  Pair blockIdx.y:
// its rows start at blockIdx.y * pair_cap.
__global__ void __launch_bounds__(256) lgr_patch_procrustes_kernel(const int* __restrict__ patch_count, const int* __restrict__ patch_off,
                                                                   int P, int min_corr, long long pair_cap, const float* __restrict__ ref_corr,
                                                                   const float* __restrict__ src_corr, const float* __restrict__ corr_scores,
                                                                   float eps, float* __restrict__ T /*[P][16]*/, int* __restrict__ valid) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.y;
    const int pl = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (pl >= P) return;
    const int p = b * P + pl;
    ref_corr += 3 * b * pair_cap; src_corr += 3 * b * pair_cap; corr_scores += b * pair_cap;
    const int c = patch_count[p], off = patch_off[b * (P + 1) + pl];
    if (c < min_corr) { if (lane == 0) valid[p] = 0; return; }
    double sw = 0.0;
    for (int e = lane; e < c; e += 32) sw += (double)fmaxf(corr_scores[off + e], 0.f);
    sw = warp_sum_d(sw);
    const double inv = 1.0 / (sw + (double)eps);
    double W = 0, S1[3] = {0, 0, 0}, S2[3] = {0, 0, 0}, Sxy[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int e = lane; e < c; e += 32) {
        const double w = (double)fmaxf(corr_scores[off + e], 0.f) * inv;
        const float* x = src_corr + 3ll * (off + e);
        const float* y = ref_corr + 3ll * (off + e);
        W += w;
        for (int a = 0; a < 3; ++a) {
            S1[a] += w * x[a]; S2[a] += w * y[a];
            for (int b = 0; b < 3; ++b) Sxy[3 * a + b] += w * (double)x[a] * (double)y[b];
        }
    }
    W = warp_sum_d(W);
    for (int a = 0; a < 3; ++a) { S1[a] = warp_sum_d(S1[a]); S2[a] = warp_sum_d(S2[a]); }
    for (int a = 0; a < 9; ++a) Sxy[a] = warp_sum_d(Sxy[a]);
    if (lane == 0) { finish_procrustes(W, S1, S2, Sxy, T + 16ll * p); valid[p] = 1; }
}

// inlier count of every valid hypothesis over ALL correspondences of its pair (local_global_registration.py:172-177)
__global__ void __launch_bounds__(256) lgr_verify_kernel(const float* __restrict__ T, const int* __restrict__ valid,
                                                         const int* __restrict__ total, long long pair_cap, const float* __restrict__ ref_corr,
                                                         const float* __restrict__ src_corr, float radius, int* __restrict__ inliers) {
    const int b = blockIdx.y;
    const int p = b * gridDim.x + blockIdx.x;
    total += b;
    ref_corr += 3 * b * pair_cap; src_corr += 3 * b * pair_cap;
    if (!valid[p]) { if (threadIdx.x == 0) inliers[p] = -1; return; }
    __shared__ float t[16];
    __shared__ int cnt;
    if (threadIdx.x < 16) t[threadIdx.x] = T[16ll * p + threadIdx.x];
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const int C = *total;
    int c = 0;
    for (int e = threadIdx.x; e < C; e += blockDim.x) {
        const float* x = src_corr + 3ll * e;
        const float* y = ref_corr + 3ll * e;
        // apply_transform: x R^T + t  (transformation.py:43)
        const float ax = fmaf(x[2], t[2], fmaf(x[1], t[1], x[0] * t[0])) + t[3];
        const float ay = fmaf(x[2], t[6], fmaf(x[1], t[5], x[0] * t[4])) + t[7];
        const float az = fmaf(x[2], t[10], fmaf(x[1], t[9], x[0] * t[8])) + t[11];
        const float dx = y[0] - ax, dy = y[1] - ay, dz = y[2] - az;
        c += (sqrtf(dx * dx + dy * dy + dz * dz) < radius) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) inliers[p] = cnt;
}

// Global refinement (single CTA): pick the best hypothesis, then num_steps weighted-SVD rounds with weights
// score * inlier(previous transform)  (local_global_registration.py:177-192).
__device__ void block_procrustes(const float* __restrict__ ref_corr, const float* __restrict__ src_corr,
                                 const float* __restrict__ corr_scores, int C, const float* Tprev /*smem or null*/, float radius,
                                 float eps, double* red /*[32][16]*/, float* Tout /*smem [16]*/) {
    // weights: score (>=0) times inlier mask under Tprev (or 1 when Tprev == nullptr)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    double acc[16];
    for (int i = 0; i < 16; ++i) acc[i] = 0.0;
    for (int e = threadIdx.x; e < C; e += blockDim.x) {
        const float* x = src_corr + 3ll * e;
        const float* y = ref_corr + 3ll * e;
        float w = fmaxf(corr_scores[e], 0.f);
        if (Tprev != nullptr) {
            const float ax = fmaf(x[2], Tprev[2], fmaf(x[1], Tprev[1], x[0] * Tprev[0])) + Tprev[3];
            const float ay = fmaf(x[2], Tprev[6], fmaf(x[1], Tprev[5], x[0] * Tprev[4])) + Tprev[7];
            const float az = fmaf(x[2], Tprev[10], fmaf(x[1], Tprev[9], x[0] * Tprev[8])) + Tprev[11];
            const float dx = y[0] - ax, dy = y[1] - ay, dz = y[2] - az;
            if (!(sqrtf(dx * dx + dy * dy + dz * dz) < radius)) w = 0.f;
        }
        const double wd = (double)w;
        acc[0] += wd;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            acc[1 + a] += wd * x[a];
            acc[4 + a] += wd * y[a];
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[7 + 3 * a + c] += wd * (double)x[a] * (double)y[c];
        }
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = warp_sum_d(acc[i]);
    if (lane == 0)
        for (int i = 0; i < 16; ++i) red[warp * 16 + i] = acc[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot[16];
        for (int i = 0; i < 16; ++i) tot[i] = 0.0;
        for (int w = 0; w < nw; ++w)
            for (int i = 0; i < 16; ++i) tot[i] += red[w * 16 + i];
        const double inv = 1.0 / (tot[0] + (double)eps);        // weights / (sum + eps)
        const double W = tot[0] * inv;
        double S1[3], S2[3], Sxy[9];
        for (int a = 0; a < 3; ++a) { S1[a] = tot[1 + a] * inv; S2[a] = tot[4 + a] * inv; }
        for (int a = 0; a < 9; ++a) Sxy[a] = tot[7 + a] * inv;
        finish_procrustes(W, S1, S2, Sxy, Tout);
    }
    __syncthreads();
}

// one CTA per pair blockIdx.x; its transform goes to Tout + blockIdx.x * t_ld
__global__ void __launch_bounds__(1024) lgr_refine_kernel(const float* __restrict__ Tpatch, const int* __restrict__ inliers, int P,
                                                          const int* __restrict__ total, long long pair_cap, const float* __restrict__ ref_corr,
                                                          const float* __restrict__ src_corr, const float* __restrict__ corr_scores,
                                                          float radius, float eps, int num_steps, float* __restrict__ Tout, int t_ld,
                                                          int* __restrict__ best_out) {
    {
        const int b = blockIdx.x;
        Tpatch += 16ll * b * P; inliers += (long long)b * P; total += b;
        ref_corr += 3 * b * pair_cap; src_corr += 3 * b * pair_cap; corr_scores += b * pair_cap;
        Tout += (long long)b * t_ld;
        if (best_out != nullptr) best_out += b;
    }
    __shared__ double red[32 * 16];
    __shared__ float Ta[16], Tb[16];
    __shared__ int best_s;
    const int C = *total;
    if (threadIdx.x == 0) {
        int best = -1, bc = -1;
        for (int p = 0; p < P; ++p)
            if (inliers[p] > bc) { bc = inliers[p]; best = p; }      // first maximum (torch.argmax) among valid patches
        best_s = (bc >= 0) ? best : -1;
        if (best_out != nullptr) *best_out = best_s;
    }
    __syncthreads();
    if (best_s >= 0) {
        if (threadIdx.x < 16) Ta[threadIdx.x] = Tpatch[16ll * best_s + threadIdx.x];
        __syncthreads();
    } else {
        // no patch with enough correspondences: global weighted SVD on the raw scores first (:179-184)
        block_procrustes(ref_corr, src_corr, corr_scores, C, nullptr, radius, eps, red, Ta);
    }
    float* cur = Ta;
    float* nxt = Tb;
    for (int s = 0; s < num_steps; ++s) {
        block_procrustes(ref_corr, src_corr, corr_scores, C, cur, radius, eps, red, nxt);
        float* t = cur; cur = nxt; nxt = t;
    }
    if (threadIdx.x < 16) Tout[threadIdx.x] = cur[threadIdx.x];
}

// generic batched weighted procrustes (modules/registration/procrustes.py:6-73): one warp per problem.  Problem b has rows
// [0, n) at row b * ld; row e is always taken by lane e % 32, so a problem's result does not depend on ld.
__device__ __forceinline__ void procrustes_warp(const float* __restrict__ src, const float* __restrict__ ref,
                                                const float* __restrict__ weights, int b, int ld, int N, float weight_thresh,
                                                float eps, float* __restrict__ T, int lane) {
    double sw = 0.0;
    for (int e = lane; e < N; e += 32) {
        float w = (weights != nullptr) ? weights[(long long)b * ld + e] : 1.f;
        if (w < weight_thresh) w = 0.f;
        sw += (double)w;
    }
    sw = warp_sum_d(sw);
    const double inv = 1.0 / (sw + (double)eps);
    double W = 0, S1[3] = {0, 0, 0}, S2[3] = {0, 0, 0}, Sxy[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int e = lane; e < N; e += 32) {
        float wf = (weights != nullptr) ? weights[(long long)b * ld + e] : 1.f;
        if (wf < weight_thresh) wf = 0.f;
        const double w = (double)wf * inv;
        const float* x = src + ((long long)b * ld + e) * 3;
        const float* y = ref + ((long long)b * ld + e) * 3;
        W += w;
        for (int a = 0; a < 3; ++a) {
            S1[a] += w * x[a]; S2[a] += w * y[a];
            for (int c = 0; c < 3; ++c) Sxy[3 * a + c] += w * (double)x[a] * (double)y[c];
        }
    }
    W = warp_sum_d(W);
    for (int a = 0; a < 3; ++a) { S1[a] = warp_sum_d(S1[a]); S2[a] = warp_sum_d(S2[a]); }
    for (int a = 0; a < 9; ++a) Sxy[a] = warp_sum_d(Sxy[a]);
    if (lane == 0) finish_procrustes(W, S1, S2, Sxy, T + 16ll * b);
}

__global__ void __launch_bounds__(256) procrustes_kernel(const float* __restrict__ src, const float* __restrict__ ref,
                                                         const float* __restrict__ weights, int B, int N, float weight_thresh,
                                                         float eps, float* __restrict__ T) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (b >= B) return;
    procrustes_warp(src, ref, weights, b, N, N, weight_thresh, eps, T, threadIdx.x & 31);
}

// the same with ragged problems: rows at or beyond counts[b] (device int32) contribute nothing
__global__ void __launch_bounds__(256) procrustes_counts_kernel(const float* __restrict__ src, const float* __restrict__ ref,
                                                                const float* __restrict__ weights, int B, int cap,
                                                                const int* __restrict__ counts, float weight_thresh, float eps,
                                                                float* __restrict__ T) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (b >= B) return;
    procrustes_warp(src, ref, weights, b, cap, min(max(counts[b], 0), cap), weight_thresh, eps, T, threadIdx.x & 31);
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_lgr_batched_workspace_bytes(int64_t n_pairs, int64_t n_patches, int64_t k, int64_t topk) {
    const size_t P = (size_t)(n_pairs * (n_patches + 1)), cap = (size_t)(k * topk * 2);
    return align_up(4 * (P + 1), 256) * 4 + align_up(4 * P * cap, 256) * 2 + align_up(64 * P, 256) + 4096;
}

// B pairs of P patches each, patches of pair b at b * P; outputs of pair b at b * (its capacity), transform at b * transform_ld.
// Correspondence outputs have capacity P*k*topk rows per pair (x2 when not mutual); num_corr[b] (device int32) = rows written.
int geob200_local_global_registration_batched(const float* ref_knn_points, const float* src_knn_points, const uint8_t* ref_knn_masks,
                                              const uint8_t* src_knn_masks, const float* log_scores, int64_t n_pairs, int64_t n_patches,
                                              int64_t k, int64_t score_ld, int64_t topk, float acceptance_radius, int mutual,
                                              float confidence_threshold, int64_t correspondence_threshold, int64_t num_refinement_steps,
                                              float* ref_corr_points, float* src_corr_points, float* corr_scores, int32_t* corr_patch,
                                              int32_t* num_corr, float* estimated_transform, int64_t transform_ld, float* patch_transforms,
                                              int32_t* patch_inliers, int32_t* best_patch, void* workspace, size_t workspace_bytes,
                                              void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= GEOB_MAX_CLOUDS / 2, "lgr_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(workspace_bytes >= geob200_lgr_batched_workspace_bytes(n_pairs, n_patches, k, topk), "lgr_batched: workspace too small");
    const int B = (int)n_pairs, P = (int)n_patches;
    GEOB_REQUIRE(P > 0 && k > 0 && k <= 256, "lgr: bad patch shape");
    GEOB_REQUIRE(topk >= 1 && topk <= 4, "lgr: topk must be in 1..4");
    GEOB_REQUIRE(score_ld == k || score_ld == k + 1, "lgr: score matrix must be (P,K,K) or (P,K+1,K+1)");
    GEOB_REQUIRE(transform_ld >= 16, "lgr: transform_ld must be >= 16");
    Arena ar(workspace, workspace_bytes);
    const int PT = B * P, K = (int)k;
    const int cap = K * (int)(mutual ? topk : 2 * topk);
    const long long pair_cap = (long long)P * cap;
    int* patch_count = ar.take<int>(PT + 1);
    int* patch_off = ar.take<int>((size_t)B * (P + 1));
    int* valid = ar.take<int>(PT + 1);
    int* inl_tmp = ar.take<int>(PT + 1);
    int* patch_ij = ar.take<int>((size_t)PT * cap);
    float* patch_score = ar.take<float>((size_t)PT * cap);
    float* T_tmp = ar.take<float>(16 * (size_t)PT);
    GEOB_REQUIRE(ar.ok(), "lgr: workspace too small");
    float* Tp = patch_transforms != nullptr ? patch_transforms : T_tmp;
    int* inl = patch_inliers != nullptr ? patch_inliers : inl_tmp;

    const size_t smem = sizeof(float) * K * (K + 1) + 2 * (size_t)K * K;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)lgr_corr_kernel<4>)) return -1;
    lgr_corr_kernel<4><<<PT, 256, smem, st>>>(log_scores, K, (int)score_ld, ref_knn_masks, src_knn_masks, (int)topk,
                                              confidence_threshold, mutual, patch_count, patch_ij, patch_score);
    lgr_offsets_kernel<<<B, 1024, 0, st>>>(patch_count, P, patch_off, num_corr);
    lgr_stack_kernel<<<dim3(P, B), 256, 0, st>>>(patch_count, patch_off, patch_ij, patch_score, K, cap, ref_knn_points, src_knn_points,
                                                 ref_corr_points, src_corr_points, corr_scores, corr_patch);
    lgr_patch_procrustes_kernel<<<dim3((P + 7) / 8, B), 256, 0, st>>>(patch_count, patch_off, P, (int)correspondence_threshold, pair_cap,
                                                                     ref_corr_points, src_corr_points, corr_scores, 1e-5f, Tp, valid);
    lgr_verify_kernel<<<dim3(P, B), 256, 0, st>>>(Tp, valid, num_corr, pair_cap, ref_corr_points, src_corr_points, acceptance_radius, inl);
    // reference: 1 procrustes with the best hypothesis' inliers + (num_refinement_steps - 1) refinements
    lgr_refine_kernel<<<B, 1024, 0, st>>>(Tp, inl, P, num_corr, pair_cap, ref_corr_points, src_corr_points, corr_scores,
                                          acceptance_radius, 1e-5f, (int)num_refinement_steps, estimated_transform, (int)transform_ld,
                                          best_patch);
    GEOB_CHECK_LAUNCH();
    count_launches(6);
    return 0;
}

int geob200_weighted_procrustes(const float* src_points, const float* ref_points, const float* weights, int64_t batch,
                                int64_t n, float weight_thresh, float eps, float* transforms, void* stream) {
    GEOB_REQUIRE(batch > 0 && n > 0, "weighted_procrustes: empty input");
    procrustes_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, (cudaStream_t)stream>>>(src_points, ref_points, weights, (int)batch,
                                                                                   (int)n, weight_thresh, eps, transforms);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_weighted_procrustes_counts(const float* src_points, const float* ref_points, const float* weights, int64_t batch,
                                       int64_t capacity, const int32_t* counts, float weight_thresh, float eps, float* transforms,
                                       void* stream) {
    GEOB_REQUIRE(batch > 0 && batch < (1ll << 31) && capacity >= 0 && capacity < (1ll << 31) / 3, "weighted_procrustes_counts: bad shape");
    GEOB_REQUIRE(counts != nullptr && transforms != nullptr, "weighted_procrustes_counts: null counts or output");
    GEOB_REQUIRE((src_points != nullptr && ref_points != nullptr) || capacity == 0, "weighted_procrustes_counts: null points");
    procrustes_counts_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, (cudaStream_t)stream>>>(src_points, ref_points, weights, (int)batch,
                                                                                         (int)capacity, counts, weight_thresh, eps,
                                                                                         transforms);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
