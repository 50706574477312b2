// Per-pair stages of the benchmark evaluation (experiments/*/eval.py) that the correspondence RANSAC and metrics kernels
// (ransac.cu) do not cover: the top-k selection of the correspondences by score, the sparse coarse precision, and the
// registration error (RRE / RTE, 3DMatch's covariance-weighted transform error, the acceptance flag).
//
// Reference: experiments/geotransformer.3dmatch.*/eval.py:125-129, 196-210 and experiments/geotransformer.kitti.*/eval.py:74-78,
//            144-146; geotransformer/utils/registration.py:17-66 (compute_registration_error), 253-281
//            (evaluate_sparse_correspondences); geotransformer/datasets/registration/threedmatch/utils.py:130-136
//            (compute_transform_error, nibabel's mat2quat).
// The reference runs these in numpy on the host, one pair at a time.  Here B pairs go in one launch (pair = blockIdx.y, or one
// CTA / thread per pair), ragged pairs in the (B, capacity, .) layout with device int32 counts, no host sync, and every
// reduction has a fixed order or counts integers, so a pair gets the same bits alone and in any batch.
#include "common.cuh"
#include "geob200.h"

namespace geob200 {

constexpr int CO_THREADS = 1024, CO_KMAX = 8192, CS_THREADS = 256, SE_THREADS = 512, RE_THREADS = 128;
constexpr size_t SE_SMEM_MAX = 96 * 1024;

__device__ __forceinline__ int be_count(const int* counts, int p, int cap) {
    return counts == nullptr ? cap : min(max(counts[p], 0), cap);
}

// ---- score order and top-k selection -------------------------------------------------------------------------------------
// 64-bit sort key of row i: ascending key = score descending, then row ascending, i.e. np.argsort(-s, kind='stable').
// -0 and +0 compare equal (numpy's comparison), every NaN sorts after every number (numpy's NaN order).
__device__ __forceinline__ unsigned long long co_key(float s, int i) {
    uint32_t u = 0xFFFFFFFFu;
    if (!isnan(s)) {
        const float f = s == 0.f ? 0.f : -s;
        u = __float_as_uint(f);
        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    }
    return ((unsigned long long)u << 32) | (uint32_t)i;
}

// One CTA per pair: order[p][0 .. min(n, kmax)) = the first rows of the order above, -1 beyond.  The keys are unique, so a radix
// select (8-bit digits, most significant first, over the pair's rows in global memory) finds the kmax-th key exactly; the keys at
// or below it (exactly kmax of them) are compacted into shared memory and bitonic-sorted there.
__global__ void __launch_bounds__(CO_THREADS) corr_order_kernel(const float* __restrict__ scores, int cap, const int* __restrict__ counts,
                                                                int kmax, int* __restrict__ order) {
    extern __shared__ unsigned long long co_buf[];      // [pow2 >= min(n, kmax)]
    __shared__ int hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_need, s_whole, s_fill;
    const int p = blockIdx.x, tid = threadIdx.x;
    const int n = be_count(counts, p, cap), m = min(n, kmax);
    scores += (long long)p * cap;
    order += (long long)p * kmax;
    unsigned long long prefix = 0;
    int shift = 64;                                      // keys with (key >> shift) <= (prefix >> shift) are selected; 64 = all
    if (n > kmax) {
        int need = kmax;
        for (int d = 7; d >= 0; --d) {
            const int sh = 8 * d;
            for (int b = tid; b < 256; b += blockDim.x) hist[b] = 0;
            __syncthreads();
            for (int i = tid; i < n; i += blockDim.x) {
                const unsigned long long c = co_key(scores[i], i);
                if (shift == 64 || (c >> shift) == (prefix >> shift)) atomicAdd(&hist[(c >> sh) & 255], 1);
            }
            __syncthreads();
            if (tid == 0) {
                int b = 0, below = 0;
                while (below + hist[b] < need) below += hist[b++];
                s_need = need - below;
                s_whole = hist[b] == need - below;
                s_prefix = prefix | ((unsigned long long)b << sh);
            }
            __syncthreads();
            need = s_need;
            prefix = s_prefix;
            shift = sh;
            const bool whole = s_whole;
            __syncthreads();
            if (whole) break;                            // the bucket is taken whole: exactly kmax keys are selected
        }
    }
    if (tid == 0) s_fill = 0;
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
        const unsigned long long c = co_key(scores[i], i);
        if (shift == 64 || (c >> shift) <= (prefix >> shift)) co_buf[atomicAdd(&s_fill, 1)] = c;
    }
    int P2 = 1;
    while (P2 < m) P2 <<= 1;
    __syncthreads();
    for (int i = m + tid; i < P2; i += blockDim.x) co_buf[i] = ~0ull;
    __syncthreads();
    for (int k = 2; k <= P2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P2; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = co_buf[i], b = co_buf[l];
                    if ((a > b) == ((i & k) == 0)) { co_buf[i] = b; co_buf[l] = a; }
                }
            }
            __syncthreads();
        }
    for (int i = tid; i < kmax; i += blockDim.x) order[i] = i < m ? (int)(uint32_t)co_buf[i] : -1;
}

// Grid (ceil(out_cap / 256), B): row i < min(n, k) of pair p = its row order[p][i] when n > k, its own row i otherwise (the
// reference selects only when there are more than k rows, and RANSAC's draws depend on the row order); zeros beyond.
__global__ void __launch_bounds__(CS_THREADS) corr_select_kernel(const float* __restrict__ ref, const float* __restrict__ src,
                                                                 const float* __restrict__ scores, int cap, const int* __restrict__ counts,
                                                                 const int* __restrict__ order, int kmax, int k, int out_cap,
                                                                 float* __restrict__ ref_out, float* __restrict__ src_out,
                                                                 float* __restrict__ score_out, int* __restrict__ count_out) {
    const int p = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = be_count(counts, p, cap), m = min(n, k);
    if (i == 0) count_out[p] = m;
    if (i >= out_cap) return;
    const long long o = (long long)p * out_cap + i;
    if (i < m) {
        const long long q = (long long)p * cap + (n <= k ? i : order[(long long)p * kmax + i]);
        for (int a = 0; a < 3; ++a) { ref_out[3 * o + a] = ref[3 * q + a]; src_out[3 * o + a] = src[3 * q + a]; }
        score_out[o] = scores[q];
    } else {
        for (int a = 0; a < 3; ++a) { ref_out[3 * o + a] = 0.f; src_out[3 * o + a] = 0.f; }
        score_out[o] = 0.f;
    }
}

// ---- sparse coarse evaluation ----------------------------------------------------------------------------------------------
template <int NV>
__device__ __forceinline__ void block_sum_u64(unsigned long long (&v)[NV], unsigned long long (*red)[32]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        if (lane == 0) red[k][warp] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        unsigned long long s = 0;
        for (int w = 0; w < nw; ++w) s += red[k][w];
        v[k] = s;
    }
    __syncthreads();
}

// One CTA per pair.  The reference assigns into dense M x N 0/1 matrices; here the gt and predicted sets are bitmaps (rows of wpr
// words, duplicates collapse), in shared memory when both fit, otherwise in the pair's slice of the workspace.  Every count is an
// exact integer and the ratios are formed in double as numpy forms them, so the three values equal numpy's bit for bit.
// out[p] = [precision, recall, hit_ratio].
__global__ void __launch_bounds__(SE_THREADS) sparse_eval_kernel(const int64_t* __restrict__ pred_ref, const int64_t* __restrict__ pred_src,
                                                                 int pred_cap, const int* __restrict__ pred_count,
                                                                 const int64_t* __restrict__ gt, int gt_cap, const int* __restrict__ gt_count,
                                                                 int m_cap, int n_cap, int wpr, uint32_t* __restrict__ gws,
                                                                 long long ws_words, double* __restrict__ out) {
    extern __shared__ uint32_t se_smem[];
    __shared__ unsigned long long red[7][32];
    const int p = blockIdx.x, tid = threadIdx.x;
    const long long words = (long long)m_cap * wpr;
    uint32_t* G = gws != nullptr ? gws + p * ws_words : se_smem;
    uint32_t* P = G + words;
    uint32_t* colG = P + words;                          // OR of the gt rows / of the positive rows
    uint32_t* colX = colG + wpr;
    for (long long w = tid; w < 2 * words + 2 * wpr; w += blockDim.x) G[w] = 0u;
    __syncthreads();
    const int ng = be_count(gt_count, p, gt_cap), np = be_count(pred_count, p, pred_cap);
    gt += 2ll * p * gt_cap;
    for (int i = tid; i < ng; i += blockDim.x) {
        const int64_t r = gt[2 * i], c = gt[2 * i + 1];
        if (r >= 0 && r < m_cap && c >= 0 && c < n_cap) atomicOr(&G[r * wpr + (c >> 5)], 1u << (c & 31));
    }
    pred_ref += (long long)p * pred_cap;
    pred_src += (long long)p * pred_cap;
    for (int i = tid; i < np; i += blockDim.x) {
        const int64_t r = pred_ref[i], c = pred_src[i];
        if (r >= 0 && r < m_cap && c >= 0 && c < n_cap) atomicOr(&P[r * wpr + (c >> 5)], 1u << (c & 31));
    }
    __syncthreads();
    // v = [gt pairs, predicted pairs, positive pairs, rows with a gt pair, rows with a positive pair, columns ditto]
    unsigned long long v[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int r = tid; r < m_cap; r += blockDim.x) {
        uint32_t any_g = 0, any_x = 0;
        for (int w = 0; w < wpr; ++w) {
            const uint32_t g = G[(long long)r * wpr + w], q = P[(long long)r * wpr + w], x = g & q;
            v[0] += __popc(g); v[1] += __popc(q); v[2] += __popc(x);
            any_g |= g; any_x |= x;
            if (g) atomicOr(&colG[w], g);
            if (x) atomicOr(&colX[w], x);
        }
        v[3] += any_g != 0u;
        v[4] += any_x != 0u;
    }
    __syncthreads();
    for (int w = tid; w < wpr; w += blockDim.x) { v[5] += __popc(colG[w]); v[6] += __popc(colX[w]); }
    block_sum_u64(v, red);
    if (tid == 0) {
        const double precision = (double)v[2] / ((double)v[1] + 1e-12);
        const double recall = (double)v[2] / ((double)v[0] + 1e-12);
        const double ref_hit = (double)v[4] / ((double)v[3] + 1e-12);
        const double src_hit = (double)v[6] / ((double)v[5] + 1e-12);
        out[3 * p] = precision;
        out[3 * p + 1] = recall;
        out[3 * p + 2] = 0.5 * (ref_hit + src_hit);
    }
}

// ---- registration error ----------------------------------------------------------------------------------------------------
// inverse of a general 4x4 (Gauss-Jordan, partial pivoting) in double; returns false when singular
__device__ bool re_inverse4(const double* A, double* X) {
    double a[4][8];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) { a[i][j] = A[4 * i + j]; a[i][4 + j] = i == j ? 1.0 : 0.0; }
    for (int c = 0; c < 4; ++c) {
        int piv = c;
        for (int r = c + 1; r < 4; ++r) if (fabs(a[r][c]) > fabs(a[piv][c])) piv = r;
        if (a[piv][c] == 0.0) return false;
        if (piv != c)
            for (int j = 0; j < 8; ++j) { const double t = a[c][j]; a[c][j] = a[piv][j]; a[piv][j] = t; }
        const double inv = 1.0 / a[c][c];
        for (int j = 0; j < 8; ++j) a[c][j] *= inv;
        for (int r = 0; r < 4; ++r)
            if (r != c) {
                const double f = a[r][c];
                for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j];
            }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) X[4 * i + j] = a[i][4 + j];
    return true;
}

// nibabel.quaternions.mat2quat: q = [w, x, y, z] = the eigenvector of the largest eigenvalue of Bar-Itzhack's symmetric K (lower
// triangle as nibabel builds it, / 3), reordered, sign-flipped so that w >= 0.  Eigenvectors by cyclic Jacobi in double.
__device__ void re_mat2quat(const double* M, double* q) {
    const double Qxx = M[0], Qyx = M[1], Qzx = M[2], Qxy = M[3], Qyy = M[4], Qzy = M[5], Qxz = M[6], Qyz = M[7], Qzz = M[8];
    double A[4][4], V[4][4];
    const double L[4][4] = {{Qxx - Qyy - Qzz, 0, 0, 0},
                            {Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0},
                            {Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0},
                            {Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz}};
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) { A[i][j] = (i >= j ? L[i][j] : L[j][i]) / 3.0; V[i][j] = i == j ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 32; ++sweep) {
        double off = 0.0;
        for (int i = 0; i < 4; ++i)
            for (int j = i + 1; j < 4; ++j) off += A[i][j] * A[i][j];
        if (off == 0.0) break;
        for (int p = 0; p < 3; ++p)
            for (int r = p + 1; r < 4; ++r) {
                const double apq = A[p][r];
                if (apq == 0.0) continue;
                const double theta = (A[r][r] - A[p][p]) / (2.0 * apq);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 4; ++k) {
                    const double akp = A[k][p], akq = A[k][r];
                    A[k][p] = c * akp - s * akq; A[k][r] = s * akp + c * akq;
                }
                for (int k = 0; k < 4; ++k) {
                    const double apk = A[p][k], aqk = A[r][k];
                    A[p][k] = c * apk - s * aqk; A[r][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 4; ++k) {
                    const double vkp = V[k][p], vkq = V[k][r];
                    V[k][p] = c * vkp - s * vkq; V[k][r] = s * vkp + c * vkq;
                }
            }
    }
    int best = 0;
    for (int i = 1; i < 4; ++i) if (A[i][i] > A[best][best]) best = i;
    q[0] = V[3][best]; q[1] = V[0][best]; q[2] = V[1][best]; q[3] = V[2][best];
    if (q[0] < 0.0) for (int i = 0; i < 4; ++i) q[i] = -q[i];
}

// One thread per pair, in double.  out[p] = [rre (deg), rte, p (NaN without a covariance), accepted].
// mode 0 (3DMatch): accepted = the pair has a covariance and p < threshold0 (the caller passes rmse_threshold^2);
// mode 1 (KITTI):   accepted = rre < threshold0 and rte < threshold1.
__global__ void __launch_bounds__(RE_THREADS) registration_error_kernel(const float* __restrict__ gt_T, int gt_ld, const float* __restrict__ est_T,
                                                                        int est_ld, const float* __restrict__ cov, const int* __restrict__ has_cov,
                                                                        int B, int mode, double thr0, double thr1, double* __restrict__ out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= B) return;
    double G[16], E[16];
    for (int e = 0; e < 16; ++e) { G[e] = gt_T[(long long)p * gt_ld + e]; E[e] = est_T[(long long)p * est_ld + e]; }
    double tr = 0.0;                                     // trace(R_est^T R_gt)
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) tr += E[4 * i + j] * G[4 * i + j];
    const double x = fmin(fmax(0.5 * (tr - 1.0), -1.0), 1.0);
    const double rre = 180.0 * acos(x) / 3.14159265358979323846;
    const double dx = G[3] - E[3], dy = G[7] - E[7], dz = G[11] - E[11];
    const double rte = sqrt(dx * dx + dy * dy + dz * dz);
    double perr = __longlong_as_double(0x7ff8000000000000ll);
    const bool cov_ok = cov != nullptr && (has_cov == nullptr || has_cov[p] != 0);
    if (cov_ok) {
        double Gi[16], Rl[16];
        if (re_inverse4(G, Gi)) {
            for (int i = 0; i < 4; ++i)
                for (int j = 0; j < 4; ++j) {
                    double s = 0.0;
                    for (int k = 0; k < 4; ++k) s += Gi[4 * i + k] * E[4 * k + j];
                    Rl[4 * i + j] = s;
                }
            const double R[9] = {Rl[0], Rl[1], Rl[2], Rl[4], Rl[5], Rl[6], Rl[8], Rl[9], Rl[10]};
            double q[4];
            re_mat2quat(R, q);
            const double er[6] = {Rl[3], Rl[7], Rl[11], q[1], q[2], q[3]};
            const float* C = cov + 36ll * p;
            double s = 0.0;
            for (int i = 0; i < 6; ++i) {
                double row = 0.0;
                for (int j = 0; j < 6; ++j) row += (double)C[6 * i + j] * er[j];
                s += er[i] * row;
            }
            perr = s / (double)C[0];
        }
    }
    const bool acc = mode == 0 ? (cov_ok && perr < thr0) : (rre < thr0 && rte < thr1);
    out[4ll * p] = rre;
    out[4ll * p + 1] = rte;
    out[4ll * p + 2] = perr;
    out[4ll * p + 3] = acc ? 1.0 : 0.0;
}

}  // namespace geob200

using namespace geob200;

extern "C" {

int geob200_corr_order_batched(const float* scores, int64_t n_pairs, int64_t capacity, const int32_t* num_corr, int64_t kmax, int32_t* order,
                               void* stream) {
    GEOB_REQUIRE(kmax >= 1 && kmax <= CO_KMAX, "corr_order: kmax must be in 1..%d", CO_KMAX);
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "corr_order: 1..65535 pairs");
    GEOB_REQUIRE(capacity >= 0 && capacity < (1ll << 31) / 3, "corr_order: bad capacity");
    GEOB_REQUIRE(scores != nullptr || capacity == 0, "corr_order: null scores");
    GEOB_REQUIRE(order != nullptr, "corr_order: null output");
    int P2 = 1;
    while (P2 < kmax) P2 <<= 1;
    const size_t smem = sizeof(unsigned long long) * (size_t)P2;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)corr_order_kernel)) return -1;
    corr_order_kernel<<<(unsigned)n_pairs, CO_THREADS, smem, (cudaStream_t)stream>>>(scores, (int)capacity, num_corr, (int)kmax, order);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_corr_select_batched(const float* ref_corr_points, const float* src_corr_points, const float* corr_scores, int64_t n_pairs,
                                int64_t capacity, const int32_t* num_corr, const int32_t* order, int64_t kmax, int64_t k,
                                float* ref_out, float* src_out, float* scores_out, int32_t* count_out, void* stream) {
    GEOB_REQUIRE(kmax >= 1 && kmax <= CO_KMAX, "corr_select: kmax must be in 1..%d", CO_KMAX);
    GEOB_REQUIRE(k >= 1 && k <= kmax, "corr_select: k must be in 1..kmax");
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "corr_select: 1..65535 pairs");
    GEOB_REQUIRE(capacity >= 0 && capacity < (1ll << 31) / 3, "corr_select: bad capacity");
    GEOB_REQUIRE((ref_corr_points != nullptr && src_corr_points != nullptr && corr_scores != nullptr) || capacity == 0,
                 "corr_select: null input");
    GEOB_REQUIRE(order != nullptr && ref_out != nullptr && src_out != nullptr && scores_out != nullptr && count_out != nullptr,
                 "corr_select: null output");
    const int out_cap = (int)(k < capacity ? k : capacity);
    const unsigned gx = (unsigned)((out_cap > 0 ? out_cap : 1) + CS_THREADS - 1) / CS_THREADS;
    corr_select_kernel<<<dim3(gx, (unsigned)n_pairs), CS_THREADS, 0, (cudaStream_t)stream>>>(
        ref_corr_points, src_corr_points, corr_scores, (int)capacity, num_corr, order, (int)kmax, (int)k, out_cap, ref_out, src_out,
        scores_out, count_out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

static size_t se_bitmap_bytes(int64_t m_cap, int64_t n_cap) {
    const size_t wpr = (size_t)((n_cap + 31) / 32);
    return 4 * (2 * (size_t)m_cap * wpr + 2 * wpr);
}

size_t geob200_sparse_correspondence_eval_batched_workspace_bytes(int64_t n_pairs, int64_t m_cap, int64_t n_cap) {
    if (n_pairs <= 0 || m_cap < 0 || n_cap < 0) return 0;
    const size_t b = se_bitmap_bytes(m_cap, n_cap);
    return b <= SE_SMEM_MAX ? 0 : (size_t)n_pairs * align_up(b, 256);
}

int geob200_sparse_correspondence_eval_batched(const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices, int64_t pred_cap,
                                               const int32_t* pred_count, const int64_t* gt_node_corr_indices, int64_t gt_cap,
                                               const int32_t* gt_count, int64_t n_pairs, int64_t m_cap, int64_t n_cap, double* out,
                                               void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "sparse_eval: 1..65535 pairs");
    GEOB_REQUIRE(m_cap >= 0 && n_cap >= 0 && m_cap * ((n_cap + 31) / 32) < (1ll << 28), "sparse_eval: bad node counts");
    GEOB_REQUIRE(pred_cap >= 0 && pred_cap < (1ll << 31) && gt_cap >= 0 && gt_cap < (1ll << 30), "sparse_eval: bad capacity");
    GEOB_REQUIRE((ref_node_corr_indices != nullptr && src_node_corr_indices != nullptr) || pred_cap == 0, "sparse_eval: null indices");
    GEOB_REQUIRE(gt_node_corr_indices != nullptr || gt_cap == 0, "sparse_eval: null gt indices");
    GEOB_REQUIRE(out != nullptr, "sparse_eval: null output");
    const size_t need = geob200_sparse_correspondence_eval_batched_workspace_bytes(n_pairs, m_cap, n_cap);
    GEOB_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need), "sparse_eval: workspace too small");
    const size_t bytes = se_bitmap_bytes(m_cap, n_cap);
    const int wpr = (int)((n_cap + 31) / 32);
    const size_t smem = need == 0 ? bytes : 0;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)sparse_eval_kernel)) return -1;
    sparse_eval_kernel<<<(unsigned)n_pairs, SE_THREADS, smem, (cudaStream_t)stream>>>(
        ref_node_corr_indices, src_node_corr_indices, (int)pred_cap, pred_count, gt_node_corr_indices, (int)gt_cap, gt_count, (int)m_cap,
        (int)n_cap, wpr, need == 0 ? nullptr : (uint32_t*)workspace, (long long)(align_up(bytes, 256) / 4), out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_registration_error_batched(const float* gt_transforms, int64_t gt_ld, const float* est_transforms, int64_t est_ld,
                                       const float* covariances, const int32_t* has_covariance, int64_t n_pairs, int mode,
                                       double threshold0, double threshold1, double* out, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs < (1ll << 31), "registration_error: bad number of pairs");
    GEOB_REQUIRE(gt_transforms != nullptr && est_transforms != nullptr && gt_ld >= 16 && est_ld >= 16, "registration_error: bad transforms");
    GEOB_REQUIRE(mode == 0 || mode == 1, "registration_error: mode must be 0 (covariance rmse) or 1 (rre / rte thresholds)");
    GEOB_REQUIRE(mode == 1 || covariances != nullptr, "registration_error: mode 0 needs covariances");
    GEOB_REQUIRE(out != nullptr, "registration_error: null output");
    registration_error_kernel<<<(unsigned)((n_pairs + RE_THREADS - 1) / RE_THREADS), RE_THREADS, 0, (cudaStream_t)stream>>>(
        gt_transforms, (int)gt_ld, est_transforms, (int)est_ld, covariances, has_covariance, (int)n_pairs, mode, threshold0, threshold1, out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
