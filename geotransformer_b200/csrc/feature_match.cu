// Exact nearest neighbour in descriptor space (any C in 1..1024; C = 3 covers point clouds) for B pairs, and the correspondence
// index lists built from it.
//
// Reference: geotransformer/utils/pointcloud.py:11-22 (get_nearest_neighbor: scipy cKDTree.query(k=1)) and
//            geotransformer/utils/registration.py:179-234 (extract_corr_indices_from_feats: plain, mutual, bilateral).
// Contract: index(q) = argmin over the support rows s of D(q, s) = sum_c (q_c - s_c)^2 in fp64, summed over c in order with every
// operation rounded on its own (no FMA), lowest index on exact ties; distance(q) = sqrt(D).  A kd-tree is a poor fit for
// C = 256 on a GPU, so the search is brute force in three passes per direction:
//   1. screen: fp32 FMA GEMM tiles give e(q, s) = (|q|^2 + |s|^2) - 2 q.s; per query row its minimum m(q);
//   2. collect: the same tiles again; every s with e(q, s) <= m(q) + band(q) goes into the row's list (first FN_CAND kept);
//   3. exact: D in fp64 for the listed candidates; a row whose list overflowed scans every support row in fp64.
// Band.  With u = 2^-24 and gamma_n = n u / (1 - n u), the fp32 dot product of C terms is off by at most gamma_C sum |q_c s_c|
// <= gamma_C (|q|^2 + |s|^2) / 2, each norm by gamma_C of itself, and the final add and subtract round twice more, so
// |e(q, s) - d(q, s)| <= 2 gamma_{C+2} (|q|^2 + |s|^2) =: err(s) for the exact distance d.  For the fp64 minimiser s* and the
// screened minimiser s': e(s*) <= d(s*) + err(s*) <= d(s') + err(s*) (+ fp64 rounding, ~2^-50 relative) <= e(s') + err(s') + err(s*),
// so band(q) = 5 (C + 2) u (|q|^2 + max_s |s|^2) covers 4 gamma_{C+2} (...) with room for the fp32 norms' own rounding and for
// 1 / (1 - n u).  The fp64 minimiser is therefore always listed (or the row overflowed and is scanned whole): the index
// contract holds by construction, whatever the screening rounds.
#include "common.cuh"
#include "feature_match.cuh"
#include "geob200.h"

namespace geob200 {

constexpr int FN_BM = 64, FN_BN = 64, FN_BK = 32, FN_THREADS = 256, FN_CAND = 8, FN_MAX_C = 1024, FN_ROWS_PER_CTA = 8;

__device__ __forceinline__ int fn_count(const int32_t* counts, int p, int cap) {
    return counts == nullptr ? cap : min(max(counts[p], 0), cap);
}

// Squared norms in fp32, one warp per row; the per-pair maximum goes to maxnorm (non-negative floats order as their bits).
__global__ void __launch_bounds__(FN_ROWS_PER_CTA * 32) fn_norms_kernel(const float* __restrict__ x, int cap, int C,
                                                                        const int32_t* __restrict__ counts, float* __restrict__ norms,
                                                                        unsigned* __restrict__ maxnorm) {
    const int p = blockIdx.y, lane = threadIdx.x & 31;
    const int r = blockIdx.x * FN_ROWS_PER_CTA + (threadIdx.x >> 5);
    if (r >= cap) return;
    const int n = fn_count(counts, p, cap);
    float v = 0.f;
    if (r < n) {
        const float* row = x + ((long long)p * cap + r) * C;
        for (int c = lane; c < C; c += 32) v = fmaf(row[c], row[c], v);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    }
    if (lane == 0) {
        norms[(long long)p * cap + r] = v;
        if (r < n) atomicMax(maxnorm + p, __float_as_uint(v));
    }
}

// Passes 1 (COLLECT = false: row minimum) and 2 (COLLECT = true: candidate lists).  Grid (ceil(cap_q / 64), B), 256 threads;
// thread (ty, tx) = (tid / 16, tid % 16) owns query rows 4 ty .. 4 ty + 3 and, per support tile, columns 4 tx .. 4 tx + 3.
template <bool COLLECT>
__global__ void __launch_bounds__(FN_THREADS) fn_screen_kernel(const float* __restrict__ Q, const float* __restrict__ S, int cap_q, int cap_s,
                                                               int C, const int32_t* __restrict__ nq_c, const int32_t* __restrict__ ns_c,
                                                               const float* __restrict__ qn, const float* __restrict__ sn,
                                                               const unsigned* __restrict__ smax, float* __restrict__ rowmin,
                                                               int* __restrict__ cand_cnt, int* __restrict__ cand) {
    __shared__ __align__(16) float qs[FN_BK][FN_BM + 4];
    __shared__ __align__(16) float ss[FN_BK][FN_BN + 4];
    const int p = blockIdx.y, tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int nq = fn_count(nq_c, p, cap_q), ns = fn_count(ns_c, p, cap_s);
    const int q0 = blockIdx.x * FN_BM;
    if (q0 >= nq || ns == 0) return;                                    // uniform over the CTA
    Q += (long long)p * cap_q * C; S += (long long)p * cap_s * C;
    qn += (long long)p * cap_q; sn += (long long)p * cap_s; rowmin += (long long)p * cap_q; cand_cnt += (long long)p * cap_q;
    cand += (long long)p * cap_q * FN_CAND;
    float qnr[4], best[4];
    double thr[4];
    const double smx = (double)__uint_as_float(smax[p]);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = q0 + 4 * ty + i;
        qnr[i] = r < nq ? qn[r] : 0.f;
        best[i] = INFINITY;
        thr[i] = -INFINITY;
        if (COLLECT && r < nq) thr[i] = (double)rowmin[r] + 5.0 * (C + 2) * 0x1p-24 * ((double)qnr[i] + smx);
    }
    for (int s0 = 0; s0 < ns; s0 += FN_BN) {
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        for (int c0 = 0; c0 < C; c0 += FN_BK) {
            __syncthreads();
#pragma unroll
            for (int e = tid; e < FN_BK * FN_BM; e += FN_THREADS) {
                const int k = e % FN_BK, m = e / FN_BK, c = c0 + k;
                qs[k][m] = (q0 + m < nq && c < C) ? Q[(long long)(q0 + m) * C + c] : 0.f;
                ss[k][m] = (s0 + m < ns && c < C) ? S[(long long)(s0 + m) * C + c] : 0.f;
            }
            __syncthreads();
#pragma unroll 8
            for (int k = 0; k < FN_BK; ++k) {
                const float4 a = *reinterpret_cast<const float4*>(&qs[k][4 * ty]);
                const float4 b = *reinterpret_cast<const float4*>(&ss[k][4 * tx]);
                const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int s = s0 + 4 * tx + j;
            if (s >= ns) continue;
            const float snj = sn[s];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float e = __fsub_rn(__fadd_rn(qnr[i], snj), __fmul_rn(2.f, acc[i][j]));
                if (!COLLECT) {
                    best[i] = fminf(best[i], e);
                } else if ((double)e <= thr[i]) {
                    const int r = q0 + 4 * ty + i;
                    const int slot = atomicAdd(cand_cnt + r, 1);
                    if (slot < FN_CAND) cand[(long long)r * FN_CAND + slot] = s;
                }
            }
        }
    }
    if (!COLLECT) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int o = 1; o < 16; o <<= 1) best[i] = fminf(best[i], __shfl_xor_sync(0xffffffffu, best[i], o));
            const int r = q0 + 4 * ty + i;
            if (tx == 0 && r < nq) rowmin[r] = best[i];
        }
    }
}

// D(q, s) of the contract: fp64, c in order, no contraction
__device__ __forceinline__ double fn_exact(const float* __restrict__ q, const float* __restrict__ s, int C) {
    double acc = 0.0;
    for (int c = 0; c < C; ++c) {
        const double t = __dsub_rn((double)q[c], (double)s[c]);
        acc = __dadd_rn(acc, __dmul_rn(t, t));
    }
    return acc;
}

// Pass 3: one warp per query row.  Rows past the count get index -1 and distance NaN; with an empty support, -1 and +inf.
__global__ void __launch_bounds__(FN_ROWS_PER_CTA * 32, 1) fn_exact_kernel(const float* __restrict__ Q, const float* __restrict__ S, int cap_q,
                                                                        int cap_s, int C, const int32_t* __restrict__ nq_c,
                                                                        const int32_t* __restrict__ ns_c, const int* __restrict__ cand_cnt,
                                                                        const int* __restrict__ cand, int64_t* __restrict__ index,
                                                                        double* __restrict__ dist) {
    const int p = blockIdx.y, lane = threadIdx.x & 31;
    const int r = blockIdx.x * FN_ROWS_PER_CTA + (threadIdx.x >> 5);
    if (r >= cap_q) return;
    const int nq = fn_count(nq_c, p, cap_q), ns = fn_count(ns_c, p, cap_s);
    const long long o = (long long)p * cap_q + r;
    if (r >= nq || ns == 0) {
        if (lane == 0) { index[o] = -1; dist[o] = r >= nq ? __longlong_as_double(0x7ff8000000000000ll) : INFINITY; }
        return;
    }
    const float* q = Q + o * C;
    S += (long long)p * cap_s * C;
    const int cnt = cand_cnt[o];
    double bd = INFINITY;
    int bi = 0x7fffffff;
    if (cnt >= 1 && cnt <= FN_CAND) {                                  // cnt == 0 only for NaN input: scan the row
        if (lane < cnt) {
            bi = cand[o * FN_CAND + lane];
            bd = fn_exact(q, S + (long long)bi * C, C);
        }
    } else {
        for (int s = lane; s < ns; s += 32) {                          // increasing s per lane: strict < keeps the lowest index
            const double d = fn_exact(q, S + (long long)s * C, C);
            if (d < bd) { bd = d; bi = s; }
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const double d = __shfl_xor_sync(0xffffffffu, bd, off);
        const int i = __shfl_xor_sync(0xffffffffu, bi, off);
        if (d < bd || (d == bd && i < bi)) { bd = d; bi = i; }
    }
    if (lane == 0) { index[o] = bi; dist[o] = __dsqrt_rn(bd); }
}

// Correspondence lists of one pair (extract_corr_indices_from_feats): mode 0 plain (ref row r <-> ref_nn[r]), 1 mutual (the rows
// r with src_nn[ref_nn[r]] == r, in increasing r), 2 bilateral (plain, then src_nn[s] <-> s for every src row s).  feat_dist is
// the descriptor distance of every listed pair in fp32.  One CTA of 1024 threads; the mutual compaction is an ordered block scan.
__global__ void __launch_bounds__(1024) fn_corr_kernel(const int64_t* __restrict__ ref_nn, const double* __restrict__ ref_dist,
                                                       const int64_t* __restrict__ src_nn, const double* __restrict__ src_dist, int n_ref,
                                                       int n_src, int mode, int64_t* __restrict__ ref_corr, int64_t* __restrict__ src_corr,
                                                       float* __restrict__ feat_dist, int32_t* __restrict__ count) {
    __shared__ int wsum[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (mode != 1) {
        for (int r = tid; r < n_ref; r += blockDim.x) {
            ref_corr[r] = r; src_corr[r] = ref_nn[r];
            if (feat_dist != nullptr) feat_dist[r] = (float)ref_dist[r];
        }
        if (mode == 2)
            for (int s = tid; s < n_src; s += blockDim.x) {
                ref_corr[n_ref + s] = src_nn[s]; src_corr[n_ref + s] = s;
                if (feat_dist != nullptr) feat_dist[n_ref + s] = (float)src_dist[s];
            }
        if (tid == 0) *count = mode == 2 ? n_ref + n_src : n_ref;
        return;
    }
    int base = 0;
    for (int c0 = 0; c0 < n_ref; c0 += blockDim.x) {
        const int r = c0 + tid;
        int f = 0;
        if (r < n_ref) {
            const int64_t s = ref_nn[r];
            f = s >= 0 && s < n_src && src_nn[s] == r;
        }
        int incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = wsum[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += v;
            }
            wsum[lane] = wi - w;                                       // exclusive prefix of the warp totals
        }
        __syncthreads();
        const int pos = base + wsum[warp] + incl - f;
        if (f) {
            ref_corr[pos] = r; src_corr[pos] = ref_nn[r];
            if (feat_dist != nullptr) feat_dist[pos] = (float)ref_dist[r];
        }
        const int last = __shfl_sync(0xffffffffu, wsum[warp] + incl, 31);
        __syncthreads();
        if (tid == blockDim.x - 1) wsum[0] = last;                    // total of this chunk
        __syncthreads();
        base += wsum[0];
        __syncthreads();
    }
    if (tid == 0) *count = base;
}

size_t feature_nn_workspace(int64_t n_pairs, int64_t cap_q, int64_t cap_s) {
    const size_t B = (size_t)(n_pairs > 0 ? n_pairs : 0), q = (size_t)(cap_q > 0 ? cap_q : 0), s = (size_t)(cap_s > 0 ? cap_s : 0);
    const size_t m = q > s ? q : s;
    return align_up(4 * B * q, 256) + align_up(4 * B * s, 256) + 2 * align_up(4 * B, 256) + 2 * align_up(4 * B * m, 256) +
           align_up(4 * B * m * FN_CAND, 256) + 256;
}

int feature_nn_launch(const float* query, const float* support, int B, int cap_q, int cap_s, int C, const int32_t* n_query,
                      const int32_t* n_support, int64_t* q_index, double* q_dist, int64_t* s_index, double* s_dist, void* workspace,
                      size_t workspace_bytes, cudaStream_t st, int* launches) {
    Arena ar(workspace, workspace_bytes);
    const int m = cap_q > cap_s ? cap_q : cap_s;
    float* qn = ar.take<float>((size_t)B * cap_q);
    float* sn = ar.take<float>((size_t)B * cap_s);
    unsigned* qmax = ar.take<unsigned>(B);
    unsigned* smax = ar.take<unsigned>(B);
    float* rowmin = ar.take<float>((size_t)B * m);
    int* cnt = ar.take<int>((size_t)B * m);
    int* cand = ar.take<int>((size_t)B * m * FN_CAND);
    GEOB_REQUIRE(ar.ok(), "feature_nn: workspace too small");
    int nl = 0;
    GEOB_CHECK_CUDA(cudaMemsetAsync(qmax, 0, 4 * (size_t)B, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(smax, 0, 4 * (size_t)B, st));
    if (cap_q > 0) { fn_norms_kernel<<<dim3((cap_q + FN_ROWS_PER_CTA - 1) / FN_ROWS_PER_CTA, B), FN_ROWS_PER_CTA * 32, 0, st>>>(query, cap_q, C, n_query, qn, qmax); ++nl; }
    if (cap_s > 0) { fn_norms_kernel<<<dim3((cap_s + FN_ROWS_PER_CTA - 1) / FN_ROWS_PER_CTA, B), FN_ROWS_PER_CTA * 32, 0, st>>>(support, cap_s, C, n_support, sn, smax); ++nl; }
    for (int dir = 0; dir < (s_index != nullptr ? 2 : 1); ++dir) {
        const float *Q = dir ? support : query, *S = dir ? query : support, *qnn = dir ? sn : qn, *snn = dir ? qn : sn;
        const int cq = dir ? cap_s : cap_q, cs = dir ? cap_q : cap_s;
        const int32_t *nq = dir ? n_support : n_query, *ns = dir ? n_query : n_support;
        const unsigned* mx = dir ? qmax : smax;
        if (cq == 0) continue;
        GEOB_CHECK_CUDA(cudaMemsetAsync(cnt, 0, 4 * (size_t)B * cq, st));
        const dim3 tiles((cq + FN_BM - 1) / FN_BM, B), rows((cq + FN_ROWS_PER_CTA - 1) / FN_ROWS_PER_CTA, B);
        fn_screen_kernel<false><<<tiles, FN_THREADS, 0, st>>>(Q, S, cq, cs, C, nq, ns, qnn, snn, mx, rowmin, cnt, cand);
        fn_screen_kernel<true><<<tiles, FN_THREADS, 0, st>>>(Q, S, cq, cs, C, nq, ns, qnn, snn, mx, rowmin, cnt, cand);
        fn_exact_kernel<<<rows, FN_ROWS_PER_CTA * 32, 0, st>>>(Q, S, cq, cs, C, nq, ns, cnt, cand, dir ? s_index : q_index, dir ? s_dist : q_dist);
        nl += 3;
    }
    GEOB_CHECK_LAUNCH();
    *launches += nl;
    return 0;
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_feature_nn_batched_workspace_bytes(int64_t n_pairs, int64_t cap_query, int64_t cap_support) {
    return feature_nn_workspace(n_pairs, cap_query, cap_support);
}

int geob200_feature_nn_batched(const float* query, const float* support, int64_t n_pairs, int64_t cap_query, int64_t cap_support,
                               int64_t channels, const int32_t* n_query, const int32_t* n_support, int64_t* query_index,
                               double* query_dist, int64_t* support_index, double* support_dist, void* workspace, size_t workspace_bytes,
                               void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "feature_nn: 1..65535 pairs");
    GEOB_REQUIRE(channels >= 1 && channels <= FN_MAX_C, "feature_nn: channels must be in 1..%d", FN_MAX_C);
    GEOB_REQUIRE(cap_query >= 0 && cap_support >= 0 && cap_query < (1ll << 28) && cap_support < (1ll << 28),
                 "feature_nn: capacities must be in 0..2^28");
    GEOB_REQUIRE((query != nullptr || cap_query == 0) && (support != nullptr || cap_support == 0), "feature_nn: null descriptors");
    GEOB_REQUIRE(query_index != nullptr && query_dist != nullptr, "feature_nn: null output");
    GEOB_REQUIRE((support_index == nullptr) == (support_dist == nullptr), "feature_nn: null output (support direction needs both arrays)");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= feature_nn_workspace(n_pairs, cap_query, cap_support),
                 "feature_nn: workspace too small");
    int nl = 0;
    const int rc = feature_nn_launch(query, support, (int)n_pairs, (int)cap_query, (int)cap_support, (int)channels, n_query, n_support,
                                     query_index, query_dist, support_index, support_dist, workspace, workspace_bytes,
                                     (cudaStream_t)stream, &nl);
    count_launches(nl);
    return rc;
}

int geob200_feature_corr_indices(const int64_t* ref_nn, const double* ref_dist, const int64_t* src_nn, const double* src_dist,
                                 int64_t n_ref, int64_t n_src, int32_t mode, int64_t* ref_corr, int64_t* src_corr, float* feat_dist,
                                 int32_t* count, void* stream) {
    GEOB_REQUIRE(mode >= 0 && mode <= 2, "feature_corr_indices: mode must be 0 (plain), 1 (mutual) or 2 (bilateral)");
    GEOB_REQUIRE(n_ref >= 0 && n_src >= 0 && n_ref + n_src < (1ll << 31), "feature_corr_indices: bad counts");
    GEOB_REQUIRE((ref_nn != nullptr && ref_dist != nullptr) || n_ref == 0, "feature_corr_indices: null ref neighbours");
    GEOB_REQUIRE(mode == 0 || (src_nn != nullptr && src_dist != nullptr) || n_src == 0, "feature_corr_indices: null src neighbours");
    GEOB_REQUIRE(ref_corr != nullptr && src_corr != nullptr && count != nullptr, "feature_corr_indices: null output");
    fn_corr_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(ref_nn, ref_dist, src_nn, src_dist, (int)n_ref, (int)n_src, mode, ref_corr, src_corr,
                                                         feat_dist, count);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
