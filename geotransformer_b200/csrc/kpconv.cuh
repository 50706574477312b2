// Pieces of the KPConv forward (kpconv.cu) that its backward (kpconv_grad.cu) recomputes with the same arithmetic.
#pragma once
#include "common.cuh"

namespace geob200 {

constexpr int KP = 15;        // kernel points of every shipped model (config.py: backbone.kernel_size)
constexpr int KP_PAD = 16;

// influence of the 15 kernel points on a neighbour at (rx, ry, rz) relative to the query point (kpconv.py:96-99)
__device__ __forceinline__ void influence15(const float* __restrict__ kp_s, float rx, float ry, float rz, float inv_dummy,
                                            float sigma, float* w) {
#pragma unroll
    for (int k = 0; k < KP; ++k) {
        const float dx = rx - kp_s[3 * k], dy = ry - kp_s[3 * k + 1], dz = rz - kp_s[3 * k + 2];
        const float sq = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        w[k] = fmaxf(1.0f - sqrtf(sq) / sigma, 0.0f);      // kpconv.py:96-99
    }
    (void)inv_dummy;
}

// cloud holding row `row` of a stacked level whose clouds start at start[0..n_clouds] (GnSeg::start)
__device__ __forceinline__ int cloud_of(const int* start, int n_clouds, int row) {
    int lo = 0, hi = n_clouds;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (start[mid] <= row) lo = mid; else hi = mid;
    }
    return lo;
}

// Pair segments of a batched level from the host row counts of its 2 n_pairs clouds (stack order [ref_1..ref_B, src_1..src_B]);
// -2 with the error set ("<what>: ...") when the counts are negative, do not add up to n_rows or n_pairs is out of range.
int make_seg(GnSeg* g, int64_t n_pairs, const int64_t* cloud_rows_h, int64_t n_rows, const char* what);

// Stage 1 of the tensor-core KPConv: pos[n] = (sum of support row n > 0), wf (n_query, 15 c_in) = the influence-weighted neighbour
// features and inv_count[m] = 1 / max(#neighbours with pos, 1).  c_in % 32 == 0.  Two launches.
void kpconv_gather(const float* s_feats, const float* q_points, const float* s_points, const long long* neighbors, int n_neighbors,
                   const float* kernel_points, float sigma, int n_support, int n_query, int c_in, unsigned char* pos, float* wf,
                   float* inv_count, cudaStream_t st);

// C[i][j] = sum_m A[m][i] * (B[m][j] * s[m]) (i < ka, j < n) over fixed 256-row chunks folded in chunk order in double
// (kpconv_grad.cu); A == nullptr: a column of ones (ka = 1, column sums), s == nullptr: ones.  `part` holds atb_bytes(M, ka, n).
size_t atb_bytes(int64_t M, int64_t ka, int64_t n);
void atb(const float* A, long long lda, const float* B, long long ldb, const float* s, int64_t M, int64_t ka, int64_t n, float* C,
         float* part, cudaStream_t st);

}  // namespace geob200
