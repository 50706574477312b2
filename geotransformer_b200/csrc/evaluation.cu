// Ground-truth superpoint correspondences (executed inside every reference forward) and the registration metrics.
//
// Reference: geotransformer/modules/registration/matching.py:231-315 (get_node_correspondences),
//            experiments/*/loss.py:95-159 (Evaluator: PIR, IR, RRE, RTE, RMSE, RR),
//            geotransformer/modules/registration/metrics.py (isotropic_transform_error).
// The reference builds (M,N) masks, a nonzero list, gathers (B,K,3) patches and a (B,K,K) distance tensor; here one CTA per
// reference superpoint walks its candidate partners with both patches in shared memory, and the metrics are one kernel.
#include "common.cuh"
#include "geob200.h"

namespace geob200 {

__device__ __forceinline__ float sqn3(float x, float y, float z) { return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)); }
__device__ __forceinline__ float sqd_mm(float ax, float ay, float az, float a2, float bx, float by, float bz, float b2) {
    const float xy = fmaf(az, bz, fmaf(ay, by, __fmul_rn(ax, bx)));          // matmul-form distance, ops/pairwise_distance.py:20-30
    return fmaxf(__fadd_rn(__fsub_rn(a2, __fmul_rn(2.0f, xy)), b2), 0.0f);
}
__device__ __forceinline__ void xform(const float* T, float x, float y, float z, float& ox, float& oy, float& oz) {
    ox = fmaf(z, T[2], fmaf(y, T[1], x * T[0])) + T[3];                      // P R^T + t (transformation.py:43)
    oy = fmaf(z, T[6], fmaf(y, T[5], x * T[4])) + T[7];
    oz = fmaf(z, T[10], fmaf(y, T[9], x * T[8])) + T[11];
}

// one warp per node: (optionally transformed) node, transformed patch points, enclosing radius over the valid patch points.
// Cloud s = blockIdx.y (rows at cl.start[s] of every array); clouds s >= t_first are transformed by T + 16 * (s - t_first).
__global__ void __launch_bounds__(256) nc_prepare_kernel(const float* __restrict__ nodes, const float* __restrict__ knn_pts,
                                                         const unsigned char* __restrict__ knn_masks, const __grid_constant__ Segs cl, int K,
                                                         const float* __restrict__ T, int t_first, float* __restrict__ nodes_out,
                                                         float* __restrict__ pts_out, float* __restrict__ max_dist, int* __restrict__ n_valid) {
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.y;
    const int m = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (m >= cl.count[s]) return;
    {
        const long long r = cl.start[s];
        nodes += 3 * r; nodes_out += 3 * r; knn_pts += 3 * r * K; pts_out += 3 * r * K; max_dist += r; n_valid += r;
        if (knn_masks != nullptr) knn_masks += r * K;
        T = (T != nullptr && s >= t_first) ? T + 16 * (s - t_first) : nullptr;
    }
    float nx = nodes[3 * m], ny = nodes[3 * m + 1], nz = nodes[3 * m + 2];
    if (T != nullptr) xform(T, nx, ny, nz, nx, ny, nz);
    float md = 0.f;
    int nv = 0;
    for (int i = lane; i < K; i += 32) {
        const float* p = knn_pts + ((long long)m * K + i) * 3;
        float px = p[0], py = p[1], pz = p[2];
        if (T != nullptr) xform(T, px, py, pz, px, py, pz);
        float* o = pts_out + ((long long)m * K + i) * 3;
        o[0] = px; o[1] = py; o[2] = pz;
        const bool ok = knn_masks == nullptr || knn_masks[(long long)m * K + i];
        const float dx = px - nx, dy = py - ny, dz = pz - nz;
        if (ok) { md = fmaxf(md, sqrtf(sqn3(dx, dy, dz))); ++nv; }
    }
    md = warp_max(md);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nv += __shfl_xor_sync(0xffffffffu, nv, o);
    if (lane == 0) {
        nodes_out[3 * m] = nx; nodes_out[3 * m + 1] = ny; nodes_out[3 * m + 2] = nz;
        max_dist[m] = md;
        n_valid[m] = nv;
    }
}

// one CTA per reference node: overlap[m][n] for every source node whose enclosing sphere intersects (matching.py:279-307)
__global__ void __launch_bounds__(256) nc_overlap_kernel(const float* __restrict__ ref_nodes, const float* __restrict__ src_nodes,
                                                         const float* __restrict__ ref_pts, const float* __restrict__ src_pts,
                                                         const unsigned char* __restrict__ ref_knn_masks,
                                                         const unsigned char* __restrict__ src_knn_masks,
                                                         const unsigned char* __restrict__ ref_masks, const unsigned char* __restrict__ src_masks,
                                                         const float* __restrict__ ref_max, const float* __restrict__ src_max,
                                                         const int* __restrict__ ref_nv, const int* __restrict__ src_nv,
                                                         const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                         const __grid_constant__ Segs NN, int K, float pos_radius,
                                                         float* __restrict__ overlap /* (M,N) per pair */) {
    // pair b = blockIdx.y: ref rows at R.start[b], src rows at Q.start[b], its (M,N) overlaps at NN.start[b]
    const int b = blockIdx.y;
    const int M = R.count[b], N = Q.count[b];
    if ((int)blockIdx.x >= M) return;
    {
        const long long r = R.start[b], q = Q.start[b];
        ref_nodes += 3 * r; ref_pts += 3 * r * K; ref_max += r; ref_nv += r;
        if (ref_knn_masks != nullptr) ref_knn_masks += r * K;
        if (ref_masks != nullptr) ref_masks += r;
        src_nodes += 3 * q; src_pts += 3 * q * K; src_max += q; src_nv += q;
        if (src_knn_masks != nullptr) src_knn_masks += q * K;
        if (src_masks != nullptr) src_masks += q;
        overlap += NN.start[b];
    }
    extern __shared__ float sm[];
    float4* rp = reinterpret_cast<float4*>(sm);         // [K] (x,y,z,|p|^2), invalid points flagged by w < 0
    float4* sp = rp + K;                                 // [K]
    int* rhit = reinterpret_cast<int*>(sp + K);          // [K]
    int* shit = rhit + K;                                // [K]
    __shared__ int tot[2];
    const int m = blockIdx.x;
    const float r2 = pos_radius * pos_radius;
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        const float* p = ref_pts + ((long long)m * K + i) * 3;
        const bool ok = ref_knn_masks == nullptr || ref_knn_masks[(long long)m * K + i];
        rp[i] = make_float4(p[0], p[1], p[2], ok ? sqn3(p[0], p[1], p[2]) : -1.f);
    }
    const bool m_ok = ref_masks == nullptr || ref_masks[m];
    const float mx = ref_nodes[3 * m], my = ref_nodes[3 * m + 1], mz = ref_nodes[3 * m + 2];
    const float m2 = sqn3(mx, my, mz);
    __syncthreads();
    for (int n = 0; n < N; ++n) {
        float ov = 0.f;
        const bool n_ok = src_masks == nullptr || src_masks[n];
        const float sx = src_nodes[3 * n], sy = src_nodes[3 * n + 1], sz = src_nodes[3 * n + 2];
        const float dist = sqrtf(sqd_mm(mx, my, mz, m2, sx, sy, sz, sqn3(sx, sy, sz)));
        const bool inter = m_ok && n_ok && (ref_max[m] + src_max[n] + pos_radius - dist > 0.f);     // block-uniform
        if (inter) {
            for (int j = threadIdx.x; j < K; j += blockDim.x) {
                const float* p = src_pts + ((long long)n * K + j) * 3;
                const bool ok = src_knn_masks == nullptr || src_knn_masks[(long long)n * K + j];
                sp[j] = make_float4(p[0], p[1], p[2], ok ? sqn3(p[0], p[1], p[2]) : -1.f);
                shit[j] = 0;
                rhit[j] = 0;
            }
            __syncthreads();
            for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
                const int i = e / K, j = e % K;
                const float4 a = rp[i], b = sp[j];
                if (a.w >= 0.f && b.w >= 0.f && sqd_mm(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w) < r2) { rhit[i] = 1; shit[j] = 1; }
            }
            __syncthreads();
            int cr = 0, cs = 0;
            for (int i = threadIdx.x; i < K; i += blockDim.x) { cr += rhit[i]; cs += shit[i]; }
            if (threadIdx.x == 0) { tot[0] = 0; tot[1] = 0; }
            __syncthreads();
            if (cr) atomicAdd(&tot[0], cr);
            if (cs) atomicAdd(&tot[1], cs);
            __syncthreads();
            ov = ((float)tot[0] / (float)ref_nv[m] + (float)tot[1] / (float)src_nv[n]) / 2.0f;
            __syncthreads();
        }
        if (threadIdx.x == 0) overlap[(long long)m * N + n] = ov;
    }
}

// ordered compaction of overlap > 0 into (C,2) indices + overlaps; one CTA per pair blockIdx.x, rows at NN.start of the pair
__global__ void __launch_bounds__(1024) nc_compact_kernel(const float* __restrict__ overlap, const __grid_constant__ Segs R,
                                                          const __grid_constant__ Segs Q, const __grid_constant__ Segs NN,
                                                          long long* __restrict__ idx, float* __restrict__ ov_out, int* __restrict__ count) {
    const int b = blockIdx.x;
    const int M = R.count[b], N = Q.count[b];
    overlap += NN.start[b]; idx += 2ll * NN.start[b]; ov_out += NN.start[b]; count += b;
    __shared__ int warp_tot[32];
    __shared__ int carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const long long total = (long long)M * N;
    for (long long base = 0; base < total; base += 4096) {                       // 4 consecutive entries per thread
        const long long t0 = base + 4ll * threadIdx.x;
        float v[4];
        int f = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            v[u] = (t0 + u < total) ? overlap[t0 + u] : 0.f;
            f += v[u] > 0.f ? 1 : 0;
        }
        int incl = f;                                                            // inclusive scan of the counts inside the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        int off = carry + incl - f;
        for (int w = 0; w < warp; ++w) off += warp_tot[w];
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (v[u] > 0.f) {
                idx[2ll * off] = (t0 + u) / N;
                idx[2ll * off + 1] = (t0 + u) % N;
                ov_out[off] = v[u];
                ++off;
            }
        __syncthreads();
        if (threadIdx.x == 0) { int s = 0; for (int w = 0; w < 32; ++w) s += warp_tot[w]; carry += s; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = carry;
}

// metrics[0..5] = PIR, IR, RRE (deg), RTE, RMSE, RR ; metrics[6] = #fine correspondences, metrics[7] = #gt node correspondences.
// mode 0 (3DMatch loss.py:133-145): RMSE of inv(T_gt) T_est x - x, RR = RMSE < rmse_threshold
// mode 1 (KITTI   loss.py:133-138): no RMSE (NaN), RR = RRE < rre_threshold and RTE < rte_threshold
// mode 2 (ModelNet loss.py:133-145): RMSE of T_est x - T_gt x, RR as in mode 1
// One CTA per pair b = blockIdx.x: gt rows at G.start[b] (G.count[b] rows), n_node_corr / n_corr rows per pair, source points at
// S0.start[b], transforms at 16 * b (gt) and b * t_ld (estimate), metrics at b * m_ld, device counts at b.
__global__ void __launch_bounds__(1024) evaluate_kernel(const long long* __restrict__ gt_idx, const float* __restrict__ gt_ov,
                                                        const __grid_constant__ Segs G, float acc_overlap,
                                                        const long long* __restrict__ ref_corr_idx, const long long* __restrict__ src_corr_idx,
                                                        int n_node_corr, const float* __restrict__ ref_corr_pts,
                                                        const float* __restrict__ src_corr_pts, int n_corr, float acc_radius,
                                                        const float* __restrict__ T_gt, const float* __restrict__ T_est, int t_ld,
                                                        const float* __restrict__ src_points, const __grid_constant__ Segs S0, int mode,
                                                        float acc_rmse, float acc_rre, float acc_rte, float* __restrict__ metrics, int m_ld,
                                                        const int* __restrict__ n_gt_dev, const int* __restrict__ n_node_corr_dev,
                                                        const int* __restrict__ n_corr_dev) {
    const int b = blockIdx.x;
    int n_gt = G.count[b];
    gt_idx += 2ll * G.start[b]; gt_ov += G.start[b];
    ref_corr_idx += (long long)b * n_node_corr; src_corr_idx += (long long)b * n_node_corr;
    ref_corr_pts += 3ll * b * n_corr; src_corr_pts += 3ll * b * n_corr;
    T_gt += 16 * b; T_est += (long long)b * t_ld;
    src_points += 3ll * S0.start[b];
    const int n_src = S0.count[b];
    metrics += (long long)b * m_ld;
    if (n_gt_dev != nullptr) n_gt_dev += b;
    if (n_node_corr_dev != nullptr) n_node_corr_dev += b;
    if (n_corr_dev != nullptr) n_corr_dev += b;
    // counts produced on the device by earlier stages (no host read-back between them and this kernel)
    if (n_gt_dev != nullptr) n_gt = *n_gt_dev;
    if (n_node_corr_dev != nullptr) n_node_corr = min(n_node_corr, *n_node_corr_dev);
    if (n_corr_dev != nullptr) n_corr = *n_corr_dev;
    __shared__ double red[32];
    __shared__ float Tg[16], Te[16], Tr[16];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < 16) { Tg[threadIdx.x] = T_gt[threadIdx.x]; Te[threadIdx.x] = T_est[threadIdx.x]; }
    __syncthreads();
    auto block_sum = [&](double v) -> double {
        v = warp_sum_d(v);
        __syncthreads();
        if (lane == 0) red[warp] = v;
        __syncthreads();
        double s = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
        return s;
    };
    const double nan = __longlong_as_double(0x7ff8000000000000LL);        // mean of an empty tensor, as torch reports it
    // PIR: fraction of predicted superpoint pairs that are ground-truth pairs with overlap > acc_overlap (loss.py:103-120)
    double hit = 0.0;
    for (int c = warp; c < n_node_corr; c += (int)(blockDim.x >> 5)) {          // one warp per predicted pair, lanes over the gt list
        const long long r = ref_corr_idx[c], s = src_corr_idx[c];
        int found = 0;
        for (int g = lane; g < n_gt; g += 32)
            if (gt_idx[2ll * g] == r && gt_idx[2ll * g + 1] == s && gt_ov[g] > acc_overlap) found = 1;
        found = __any_sync(0xffffffffu, found);
        if (lane == 0) hit += found;
    }
    const double hits = block_sum(hit);
    const double pir = n_node_corr > 0 ? hits / n_node_corr : nan;
    // IR (loss.py:123-130)
    double inl = 0.0;
    for (int c = threadIdx.x; c < n_corr; c += blockDim.x) {
        float x, y, z;
        xform(Tg, src_corr_pts[3ll * c], src_corr_pts[3ll * c + 1], src_corr_pts[3ll * c + 2], x, y, z);
        const float dx = ref_corr_pts[3ll * c] - x, dy = ref_corr_pts[3ll * c + 1] - y, dz = ref_corr_pts[3ll * c + 2] - z;
        inl += (sqrtf(sqn3(dx, dy, dz)) < acc_radius) ? 1.0 : 0.0;
    }
    const double inls = block_sum(inl);
    const double ir = n_corr > 0 ? inls / n_corr : nan;
    // realignment transform inv(T_gt) . T_est (T_gt is rigid: inverse = [R^T, -R^T t])
    if (threadIdx.x == 0) {
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) {
                double a = 0.0;
                for (int k = 0; k < 3; ++k) a += (double)Tg[4 * k + i] * Te[4 * k + j];
                Tr[4 * i + j] = (float)a;
            }
            double b = 0.0;
            for (int k = 0; k < 3; ++k) b += (double)Tg[4 * k + i] * ((double)Te[4 * k + 3] - Tg[4 * k + 3]);
            Tr[4 * i + 3] = (float)b;
        }
    }
    __syncthreads();
    double se = 0.0;
    if (mode != 1) {
        for (int p = threadIdx.x; p < n_src; p += blockDim.x) {
            const float px = src_points[3ll * p], py = src_points[3ll * p + 1], pz = src_points[3ll * p + 2];
            float x, y, z, gx = px, gy = py, gz = pz;
            if (mode == 0) {
                xform(Tr, px, py, pz, x, y, z);
            } else {
                xform(Te, px, py, pz, x, y, z);
                xform(Tg, px, py, pz, gx, gy, gz);
            }
            se += sqrtf(sqn3(x - gx, y - gy, z - gz));
        }
    }
    const double ses = block_sum(se);
    const double rmse = mode == 1 ? nan : (n_src > 0 ? ses / n_src : nan);
    if (threadIdx.x == 0) {
        // isotropic errors in fp32 like metrics.py:47-82: RRE = acos((tr(R_est^T R_gt) - 1) / 2) in degrees, RTE = |t_gt - t_est|
        float tr = 0.f;
        for (int i = 0; i < 3; ++i) {
            float d = 0.f;
            for (int k = 0; k < 3; ++k) d = fmaf(Te[4 * k + i], Tg[4 * k + i], d);
            tr += d;
        }
        float x = 0.5f * (tr - 1.0f);
        x = fminf(fmaxf(x, -1.0f), 1.0f);
        const float rre = 180.0f * acosf(x) / 3.14159265358979323846f;
        const float dtx = Tg[3] - Te[3], dty = Tg[7] - Te[7], dtz = Tg[11] - Te[11];
        const float rte = sqrtf(sqn3(dtx, dty, dtz));
        metrics[0] = (float)pir;
        metrics[1] = (float)ir;
        metrics[2] = rre;
        metrics[3] = rte;
        metrics[4] = (float)rmse;
        metrics[5] = mode == 0 ? ((float)rmse < acc_rmse ? 1.0f : 0.0f) : ((rre < acc_rre && rte < acc_rte) ? 1.0f : 0.0f);
        metrics[6] = (float)n_corr;
        metrics[7] = (float)n_gt;
    }
}

// ---------------------------------------------------------------------------------------------------- validation losses
// OverallLoss (experiments/<exp>/loss.py:10-92, modules/loss/circle_loss.py:44-86) as the reference evaluates it in val_step:
// values only, no gradients.  Every reduction runs in a fixed order (no atomics), so a pair gets the same bits alone and in a batch.

// deterministic block reduction over 256 threads: warp tree, then warp 0..7 in order
template <typename T, typename Op>
__device__ __forceinline__ T block_reduce_256(T v, Op op, T* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    T s = red[0];
    for (int w = 1; w < 8; ++w) s = op(s, red[w]);
    return s;
}

// d[i][j] = sqrt(clamp(2 - 2 <f_i, g_j>, 0)) for every (ref i, src j) of pair p = blockIdx.y (ALL superpoints: the loss applies no
// node mask), o[i][j] = 0.  One CTA per ref row, one warp per entry (lane-strided fmaf + warp_sum, as spm_scores_kernel).
__global__ void __launch_bounds__(256) closs_dist_kernel(const float* __restrict__ fr, const float* __restrict__ fs, int C,
                                                         const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                         const __grid_constant__ Segs NN, float* __restrict__ d, float* __restrict__ o) {
    extern __shared__ float a[];            // [C]
    const int p = blockIdx.y, i = blockIdx.x;
    const int M = R.count[p], N = Q.count[p];
    if (i >= M) return;
    fr += ((long long)R.start[p] + i) * C;
    fs += (long long)Q.start[p] * C;
    d += NN.start[p] + (long long)i * N;
    o += NN.start[p] + (long long)i * N;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = threadIdx.x; c < C; c += blockDim.x) a[c] = fr[c];
    __syncthreads();
    for (int j = warp; j < N; j += 8) {
        const float* b = fs + (long long)j * C;
        float x = 0.f;
        for (int c = lane; c < C; c += 32) x = fmaf(a[c], b[c], x);
        x = warp_sum(x);
        if (lane == 0) {
            d[j] = sqrtf(fmaxf(__fsub_rn(2.0f, __fmul_rn(2.0f, x)), 0.0f));
            o[j] = 0.f;
        }
    }
}

// o[i][j] = overlap of the first count[p] ground-truth rows of pair p (rows at NN.start[p])
__global__ void __launch_bounds__(256) closs_scatter_kernel(const long long* __restrict__ gt_idx, const float* __restrict__ gt_ov,
                                                            const int* __restrict__ count, const __grid_constant__ Segs Q,
                                                            const __grid_constant__ Segs NN, float* __restrict__ o) {
    const int p = blockIdx.y;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(count[p], NN.count[p]);
    if (g >= n) return;
    gt_idx += 2ll * NN.start[p]; gt_ov += NN.start[p];
    o[NN.start[p] + gt_idx[2ll * g] * Q.count[p] + gt_idx[2ll * g + 1]] = gt_ov[g];
}

struct CircleParams {
    float pos_margin, neg_margin, pos_optimal, neg_optimal, log_scale, pos_overlap;
};

// one CTA per row (blockIdx.z = 0: ref superpoint i over all j) or column (z = 1: src superpoint j over all i) of pair blockIdx.y:
// both logsumexps (max subtracted first), loss = softplus(Lp + Ln) / log_scale and kept = (has a positive and a negative).
// Weight-0 entries stay in the sums (exp(0) = 1), as in the reference.  Results at the row's / column's cloud offset.
__global__ void __launch_bounds__(256) closs_lse_kernel(const float* __restrict__ d, const float* __restrict__ o,
                                                        const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                        const __grid_constant__ Segs NN, CircleParams cp, float* __restrict__ ell_r,
                                                        unsigned char* __restrict__ kept_r, float* __restrict__ ell_c,
                                                        unsigned char* __restrict__ kept_c) {
    __shared__ float redf[8];
    __shared__ int redi[8];
    const int p = blockIdx.y, col = blockIdx.z;
    const int M = R.count[p], N = Q.count[p];
    const int line = blockIdx.x;
    if (line >= (col ? N : M)) return;
    const int len = col ? M : N;
    const long long base = NN.start[p] + (col ? line : (long long)line * N);
    const long long step = col ? N : 1;
    auto logits = [&](int e, float& lp, float& ln, int& pos, int& neg) {
        const float dv = d[base + e * step], ov = o[base + e * step];
        pos = ov > cp.pos_overlap;
        neg = ov == 0.f;
        const float wp = pos ? __fmul_rn(fmaxf(__fsub_rn(dv, cp.pos_optimal), 0.f), sqrtf(ov)) : 0.f;
        const float wn = neg ? fmaxf(__fsub_rn(cp.neg_optimal, dv), 0.f) : 0.f;
        lp = __fmul_rn(__fmul_rn(cp.log_scale, __fsub_rn(dv, cp.pos_margin)), wp);
        ln = __fmul_rn(__fmul_rn(cp.log_scale, __fsub_rn(cp.neg_margin, dv)), wn);
    };
    float mp = -INFINITY, mn = -INFINITY;
    int np_ = 0, nn_ = 0;
    for (int e = threadIdx.x; e < len; e += blockDim.x) {
        float lp, ln;
        int pos, neg;
        logits(e, lp, ln, pos, neg);
        mp = fmaxf(mp, lp); mn = fmaxf(mn, ln);
        np_ |= pos; nn_ |= neg;
    }
    auto fmax_op = [](float x, float y) { return fmaxf(x, y); };
    auto fadd_op = [](float x, float y) { return x + y; };
    auto ior_op = [](int x, int y) { return x | y; };
    mp = block_reduce_256(mp, fmax_op, redf);
    mn = block_reduce_256(mn, fmax_op, redf);
    const int has = block_reduce_256(np_ | (nn_ << 1), ior_op, redi);
    float sp = 0.f, sn = 0.f;
    for (int e = threadIdx.x; e < len; e += blockDim.x) {
        float lp, ln;
        int pos, neg;
        logits(e, lp, ln, pos, neg);
        sp += expf(lp - mp);
        sn += expf(ln - mn);
    }
    sp = block_reduce_256(sp, fadd_op, redf);
    sn = block_reduce_256(sn, fadd_op, redf);
    if (threadIdx.x == 0) {
        const float x = (mp + logf(sp)) + (mn + logf(sn));
        const float sp1 = x > 20.f ? x : log1pf(expf(x));            // torch softplus: linear above threshold 20
        const float l = sp1 / cp.log_scale;
        const long long r = (col ? Q.start[p] : R.start[p]) + line;
        (col ? ell_c : ell_r)[r] = l;
        (col ? kept_c : kept_r)[r] = has == 3;
    }
}

// one warp per pair: c_loss = (mean of the kept rows + mean of the kept columns) / 2 (NaN for an empty selection) -> out[p * ld + 1]
__global__ void __launch_bounds__(32) closs_finalize_kernel(const float* __restrict__ ell_r, const unsigned char* __restrict__ kept_r,
                                                            const float* __restrict__ ell_c, const unsigned char* __restrict__ kept_c,
                                                            const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                            float* __restrict__ out, long long ld) {
    const int p = blockIdx.x, lane = threadIdx.x;
    double m[2];
    for (int side = 0; side < 2; ++side) {
        const float* ell = side ? ell_c : ell_r;
        const unsigned char* kept = side ? kept_c : kept_r;
        const int s0 = side ? Q.start[p] : R.start[p], n = side ? Q.count[p] : R.count[p];
        double s = 0.0, k = 0.0;
        for (int i = lane; i < n; i += 32)
            if (kept[s0 + i]) { s += ell[s0 + i]; k += 1.0; }
        s = warp_sum_d(s);
        k = warp_sum_d(k);
        m[side] = (float)(s / k);              // 0 / 0 = NaN: the mean of an empty selection
    }
    if (lane == 0) out[p * ld + 1] = __fdiv_rn(__fadd_rn((float)m[0], (float)m[1]), 2.0f);
}

// FineMatchingLoss, one CTA per patch q of pair p = blockIdx.y (patch rows at p * P + q): ground-truth labels of the (K+1)^2
// Sinkhorn block (point pairs closer than the radius after the gt transform, slack row / column for unmatched valid points);
// partial[p * P + q] = (sum of the labelled scores, #labels).  Scores are read only where a label is set.
template <int K>
__global__ void __launch_bounds__(256) floss_patch_kernel(const float* __restrict__ ref_pts, const float* __restrict__ src_pts,
                                                          const unsigned char* __restrict__ ref_masks,
                                                          const unsigned char* __restrict__ src_masks, const float* __restrict__ scores,
                                                          const float* __restrict__ T, int P, const int* __restrict__ count, float r2,
                                                          double* __restrict__ psum, int* __restrict__ pcnt) {
    __shared__ float4 rp[K], sp[K];              // (x, y, z, |p|^2), w < 0 = invalid point
    __shared__ int rhit[K], shit[K];
    __shared__ double redd[8];
    __shared__ int redi[8];
    __shared__ float Tm[16];
    const int p = blockIdx.y, q = blockIdx.x;
    const long long patch = (long long)p * P + q;
    const bool live = count == nullptr || q < count[p];
    if (threadIdx.x < 16) Tm[threadIdx.x] = T[16 * p + threadIdx.x];
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        const float* a = ref_pts + (patch * K + i) * 3;
        const float* b = src_pts + (patch * K + i) * 3;
        const bool ra = live && ref_masks[patch * K + i], sa = live && src_masks[patch * K + i];
        float x, y, z;
        xform(Tm, b[0], b[1], b[2], x, y, z);
        rp[i] = make_float4(a[0], a[1], a[2], ra ? sqn3(a[0], a[1], a[2]) : -1.f);
        sp[i] = make_float4(x, y, z, sa ? sqn3(x, y, z) : -1.f);
        rhit[i] = 0;
        shit[i] = 0;
    }
    __syncthreads();
    const float* S = scores + patch * (K + 1) * (K + 1);
    double s = 0.0;
    int n = 0;
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
        const int i = e / K, j = e % K;
        const float4 a = rp[i], b = sp[j];
        if (a.w >= 0.f && b.w >= 0.f && sqd_mm(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w) < r2) {
            rhit[i] = 1;
            shit[j] = 1;
            s += S[i * (K + 1) + j];
            ++n;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        if (rp[i].w >= 0.f && !rhit[i]) { s += S[i * (K + 1) + K]; ++n; }
        if (sp[i].w >= 0.f && !shit[i]) { s += S[K * (K + 1) + i]; ++n; }
    }
    s = block_reduce_256(s, [](double x, double y) { return x + y; }, redd);
    n = block_reduce_256(n, [](int x, int y) { return x + y; }, redi);
    if (threadIdx.x == 0) { psum[patch] = s; pcnt[patch] = n; }
}

// one warp per pair: f_loss = -(sum of the labelled scores / #labels) over all patches of the pair -> out[p * ld + 2]; with weights
// also loss = w_c * out[p * ld + 1] + w_f * f_loss -> out[p * ld + 0]
__global__ void __launch_bounds__(32) floss_finalize_kernel(const double* __restrict__ psum, const int* __restrict__ pcnt, int P,
                                                            int with_total, float w_c, float w_f, float* __restrict__ out, long long ld) {
    const int p = blockIdx.x, lane = threadIdx.x;
    double s = 0.0, k = 0.0;
    for (int q = lane; q < P; q += 32) { s += psum[(long long)p * P + q]; k += pcnt[(long long)p * P + q]; }
    s = warp_sum_d(s);
    k = warp_sum_d(k);
    if (lane == 0) {
        const float f = -(float)(s / k);
        out[p * ld + 2] = f;
        if (with_total) out[p * ld] = __fadd_rn(__fmul_rn(w_c, out[p * ld + 1]), __fmul_rn(w_f, f));
    }
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_node_correspondences_workspace_bytes(int64_t n_ref, int64_t n_src, int64_t k) {
    const size_t m = (size_t)n_ref, n = (size_t)n_src, kk = (size_t)k;
    return align_up(12 * m, 256) + align_up(12 * n, 256) + align_up(12 * m * kk, 256) + align_up(12 * n * kk, 256) + 2 * align_up(4 * m, 256) +
           2 * align_up(4 * n, 256) + align_up(4 * m * n, 256) + 256;
}

size_t geob200_node_correspondences_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t k) {
    return geob200_node_correspondences_workspace_bytes(n_rows, 0, k) + align_up(4 * (size_t)n_products, 256);
}

static int nc_overlap_compact(const float* rn, const float* sn, const float* rp, const float* sp, const uint8_t* ref_knn_masks,
                              const uint8_t* src_knn_masks, const uint8_t* ref_masks, const uint8_t* src_masks, const float* rmax,
                              const float* smax, const int* rnv, const int* snv, const Segs& R, const Segs& Q, int64_t k, float pos_radius,
                              float* overlap, int64_t* corr_indices, float* corr_overlaps, int32_t* count, cudaStream_t st) {
    Segs NN;
    if (segs_products(&NN, R, Q)) return -1;
    const size_t smem = (size_t)k * (2 * sizeof(float4) + 2 * sizeof(int));
    if (R.max > 0)
        nc_overlap_kernel<<<dim3((unsigned)R.max, R.n), 256, smem, st>>>(rn, sn, rp, sp, ref_knn_masks, src_knn_masks, ref_masks, src_masks,
                                                                        rmax, smax, rnv, snv, R, Q, NN, (int)k, pos_radius, overlap);
    nc_compact_kernel<<<R.n, 1024, 0, st>>>(overlap, R, Q, NN, (long long*)corr_indices, corr_overlaps, count);
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

// corr_indices (n_ref*n_src, 2) int64 capacity, corr_overlaps (n_ref*n_src) capacity; *count = rows written (row-major order)
int geob200_node_correspondences(const float* ref_nodes, const float* src_nodes, const float* ref_knn_points, const float* src_knn_points,
                                 const uint8_t* ref_masks, const uint8_t* src_masks, const uint8_t* ref_knn_masks,
                                 const uint8_t* src_knn_masks, int64_t n_ref, int64_t n_src, int64_t k, const float* transform,
                                 float pos_radius, int64_t* corr_indices, float* corr_overlaps, int32_t* count, void* workspace,
                                 size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_ref > 0 && n_src > 0 && k > 0 && k <= 1024, "node_correspondences: bad shape");
    GEOB_REQUIRE(workspace_bytes >= geob200_node_correspondences_workspace_bytes(n_ref, n_src, k), "node_correspondences: workspace too small");
    Arena ar(workspace, workspace_bytes);
    float* rn = ar.take<float>(3 * n_ref);
    float* sn = ar.take<float>(3 * n_src);
    float* rp = ar.take<float>(3 * n_ref * k);
    float* sp = ar.take<float>(3 * n_src * k);
    float* rmax = ar.take<float>(n_ref);
    float* smax = ar.take<float>(n_src);
    int* rnv = ar.take<int>(n_ref);
    int* snv = ar.take<int>(n_src);
    float* overlap = ar.take<float>((size_t)n_ref * n_src);
    GEOB_REQUIRE(ar.ok(), "node_correspondences: workspace accounting error");
    const Segs R = segs_one(n_ref), Q = segs_one(n_src);
    nc_prepare_kernel<<<dim3((unsigned)((n_ref + 7) / 8), 1), 256, 0, st>>>(ref_nodes, ref_knn_points, ref_knn_masks, R, (int)k, nullptr, 0,
                                                                          rn, rp, rmax, rnv);
    nc_prepare_kernel<<<dim3((unsigned)((n_src + 7) / 8), 1), 256, 0, st>>>(src_nodes, src_knn_points, src_knn_masks, Q, (int)k, transform, 0,
                                                                          sn, sp, smax, snv);
    count_launches(2);
    return nc_overlap_compact(rn, sn, rp, sp, ref_knn_masks, src_knn_masks, ref_masks, src_masks, rmax, smax, rnv, snv, R, Q, k, pos_radius,
                              overlap, corr_indices, corr_overlaps, count, st);
}

int geob200_node_correspondences_batched(const float* nodes, const float* knn_points, const uint8_t* node_masks, const uint8_t* knn_masks,
                                         int64_t n_pairs, const int64_t* cloud_nodes, int64_t k, const float* transforms, float pos_radius,
                                         int64_t* corr_indices, float* corr_overlaps, int32_t* count, void* workspace, size_t workspace_bytes,
                                         void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "node_correspondences_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(k > 0 && k <= 1024, "node_correspondences: bad shape");
    Segs cl, NN;
    if (segs_from_counts(&cl, 2 * n_pairs, cloud_nodes)) return -1;
    const int B = (int)n_pairs;
    const Segs R = segs_range(cl, 0, B), Q = segs_range(cl, B, B);
    if (segs_products(&NN, R, Q)) return -1;
    const int64_t rows = (int64_t)cl.start[2 * B - 1] + cl.count[2 * B - 1];
    const int64_t nn = (int64_t)NN.start[B - 1] + NN.count[B - 1];
    GEOB_REQUIRE(workspace_bytes >= geob200_node_correspondences_batched_workspace_bytes(rows, nn, k),
                 "node_correspondences_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    float* cn = ar.take<float>(3 * rows);
    float* cp = ar.take<float>(3 * rows * k);
    float* cmax = ar.take<float>(rows);
    int* cnv = ar.take<int>(rows);
    float* overlap = ar.take<float>(nn);
    GEOB_REQUIRE(ar.ok(), "node_correspondences: workspace accounting error");
    nc_prepare_kernel<<<dim3((unsigned)((cl.max + 7) / 8 > 0 ? (cl.max + 7) / 8 : 1), 2 * B), 256, 0, st>>>(
        nodes, knn_points, knn_masks, cl, (int)k, transforms, B, cn, cp, cmax, cnv);
    count_launches(1);
    return nc_overlap_compact(cn, cn, cp, cp, knn_masks, knn_masks, node_masks, node_masks, cmax, cmax, cnv, cnv, R, Q, k, pos_radius,
                              overlap, corr_indices, corr_overlaps, count, st);
}

static int evaluate_impl(const int64_t* gt_idx, const float* gt_ov, const Segs& G, const int32_t* n_gt_dev, float acceptance_overlap,
                         const int64_t* ref_idx, const int64_t* src_idx, int64_t n_node_corr, const int32_t* n_node_corr_dev,
                         const float* ref_pts, const float* src_pts, int64_t n_corr, const int32_t* n_corr_dev, float acceptance_radius,
                         const float* gt_transform, const float* est_transform, int64_t transform_ld, const float* src_points,
                         const Segs& S0, int mode, float rmse_threshold, float rre_threshold, float rte_threshold, float* metrics,
                         int64_t metrics_ld, cudaStream_t st) {
    GEOB_REQUIRE(mode >= 0 && mode <= 2, "evaluate: mode must be 0 (3DMatch), 1 (KITTI) or 2 (ModelNet)");
    evaluate_kernel<<<G.n, 1024, 0, st>>>((const long long*)gt_idx, gt_ov, G, acceptance_overlap, (const long long*)ref_idx,
                                          (const long long*)src_idx, (int)n_node_corr, ref_pts, src_pts, (int)n_corr, acceptance_radius,
                                          gt_transform, est_transform, (int)transform_ld, src_points, S0, mode, rmse_threshold, rre_threshold,
                                          rte_threshold, metrics, (int)metrics_ld, n_gt_dev, n_node_corr_dev, n_corr_dev);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_evaluate(const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps, int64_t n_gt, float acceptance_overlap,
                     const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices, int64_t n_node_corr,
                     const float* ref_corr_points, const float* src_corr_points, int64_t n_corr, float acceptance_radius,
                     const float* gt_transform, const float* est_transform, const float* src_points, int64_t n_src_points, int mode,
                     float rmse_threshold, float rre_threshold, float rte_threshold, float* metrics, void* stream) {
    return geob200_evaluate_counts(gt_node_corr_indices, gt_node_corr_overlaps, n_gt, nullptr, acceptance_overlap, ref_node_corr_indices,
                                   src_node_corr_indices, n_node_corr, nullptr, ref_corr_points, src_corr_points, n_corr, nullptr,
                                   acceptance_radius, gt_transform, est_transform, src_points, n_src_points, mode, rmse_threshold,
                                   rre_threshold, rte_threshold, metrics, stream);
}

int geob200_evaluate_counts(const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps, int64_t n_gt, const int32_t* n_gt_dev,
                            float acceptance_overlap, const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices,
                            int64_t n_node_corr, const int32_t* n_node_corr_dev, const float* ref_corr_points, const float* src_corr_points,
                            int64_t n_corr, const int32_t* n_corr_dev, float acceptance_radius, const float* gt_transform,
                            const float* est_transform, const float* src_points, int64_t n_src_points, int mode, float rmse_threshold,
                            float rre_threshold, float rte_threshold, float* metrics, void* stream) {
    return evaluate_impl(gt_node_corr_indices, gt_node_corr_overlaps, segs_one(n_gt), n_gt_dev, acceptance_overlap, ref_node_corr_indices,
                         src_node_corr_indices, n_node_corr, n_node_corr_dev, ref_corr_points, src_corr_points, n_corr, n_corr_dev,
                         acceptance_radius, gt_transform, est_transform, 16, src_points, segs_one(n_src_points), mode, rmse_threshold,
                         rre_threshold, rte_threshold, metrics, 8, (cudaStream_t)stream);
}

int geob200_evaluate_batched(const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps, const int32_t* n_gt_dev,
                             float acceptance_overlap, const int64_t* ref_node_corr_indices, const int64_t* src_node_corr_indices,
                             int64_t n_node_corr, const int32_t* n_node_corr_dev, const float* ref_corr_points, const float* src_corr_points,
                             int64_t n_corr, const int32_t* n_corr_dev, float acceptance_radius, const float* gt_transforms,
                             const float* est_transforms, int64_t transform_ld, const float* points, int64_t n_pairs, const int64_t* cloud_nodes,
                             const int64_t* cloud_points, int mode, float rmse_threshold, float rre_threshold, float rte_threshold,
                             float* metrics, int64_t metrics_ld, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "evaluate_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(transform_ld >= 16 && metrics_ld >= 8, "evaluate_batched: transform_ld >= 16 and metrics_ld >= 8 required");
    Segs cl, pt, G;
    if (segs_from_counts(&cl, 2 * n_pairs, cloud_nodes) || segs_from_counts(&pt, 2 * n_pairs, cloud_points)) return -1;
    const int B = (int)n_pairs;
    if (segs_products(&G, segs_range(cl, 0, B), segs_range(cl, B, B))) return -1;
    return evaluate_impl(gt_node_corr_indices, gt_node_corr_overlaps, G, n_gt_dev, acceptance_overlap, ref_node_corr_indices,
                         src_node_corr_indices, n_node_corr, n_node_corr_dev, ref_corr_points, src_corr_points, n_corr, n_corr_dev,
                         acceptance_radius, gt_transforms, est_transforms, transform_ld, points, segs_range(pt, B, B), mode, rmse_threshold,
                         rre_threshold, rte_threshold, metrics, metrics_ld, (cudaStream_t)stream);
}

size_t geob200_coarse_matching_loss_batched_workspace_bytes(int64_t n_rows, int64_t n_products) {
    const size_t r = (size_t)n_rows, nn = (size_t)n_products;
    return 2 * align_up(4 * nn, 256) + align_up(4 * r, 256) + align_up(r, 256) + 256;
}

int geob200_coarse_matching_loss_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs,
                                         const int64_t* cloud_nodes, const int64_t* gt_node_corr_indices, const float* gt_node_corr_overlaps,
                                         const int32_t* gt_count, float positive_margin, float negative_margin, float positive_optimal,
                                         float negative_optimal, float log_scale, float positive_overlap, float* out, int64_t out_ld,
                                         void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "coarse_matching_loss_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(channels > 0 && channels <= 8192, "coarse_matching_loss_batched: 1..8192 channels");
    GEOB_REQUIRE(log_scale > 0.f, "coarse_matching_loss_batched: log_scale must be positive");
    GEOB_REQUIRE(out_ld >= 3, "coarse_matching_loss_batched: out_ld >= 3 required");
    GEOB_REQUIRE(gt_count != nullptr, "coarse_matching_loss_batched: gt_count (device int32, one per pair) is required");
    for (int64_t c = 0; c < 2 * n_pairs; ++c) GEOB_REQUIRE(cloud_nodes[c] >= 0, "coarse_matching_loss_batched: negative node count");
    const int B = (int)n_pairs;
    Segs R, Q, NN;
    if (segs_from_counts(&R, B, cloud_nodes) || segs_from_counts(&Q, B, cloud_nodes + B) || segs_products(&NN, R, Q)) return -1;
    const int64_t rows = (int64_t)R.start[B - 1] + R.count[B - 1] + Q.start[B - 1] + Q.count[B - 1];
    const int64_t nn = (int64_t)NN.start[B - 1] + NN.count[B - 1];
    GEOB_REQUIRE(workspace_bytes >= geob200_coarse_matching_loss_batched_workspace_bytes(rows, nn),
                 "coarse_matching_loss_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    float* d = ar.take<float>(nn);
    float* o = ar.take<float>(nn);
    float* ell = ar.take<float>(rows);
    unsigned char* kept = ar.take<unsigned char>(rows);
    GEOB_REQUIRE(ar.ok(), "coarse_matching_loss_batched: workspace accounting error");
    float* ell_c = ell + R.start[B - 1] + R.count[B - 1];
    unsigned char* kept_c = kept + R.start[B - 1] + R.count[B - 1];
    const CircleParams cp{positive_margin, negative_margin, positive_optimal, negative_optimal, log_scale, positive_overlap};
    int n_launch = 1;
    if (R.max > 0 && Q.max > 0) {
        closs_dist_kernel<<<dim3((unsigned)R.max, B), 256, channels * sizeof(float), st>>>(ref_feats, src_feats, (int)channels, R, Q, NN, d, o);
        closs_scatter_kernel<<<dim3((unsigned)((NN.max + 255) / 256), B), 256, 0, st>>>((const long long*)gt_node_corr_indices,
                                                                                        gt_node_corr_overlaps, gt_count, Q, NN, o);
        n_launch += 2;
    }
    if (R.max > 0 || Q.max > 0) {
        closs_lse_kernel<<<dim3((unsigned)(R.max > Q.max ? R.max : Q.max), B, 2), 256, 0, st>>>(d, o, R, Q, NN, cp, ell, kept, ell_c, kept_c);
        n_launch += 1;
    }
    closs_finalize_kernel<<<B, 32, 0, st>>>(ell, kept, ell_c, kept_c, R, Q, out, (long long)out_ld);
    GEOB_CHECK_LAUNCH();
    count_launches(n_launch);
    return 0;
}

size_t geob200_fine_matching_loss_batched_workspace_bytes(int64_t n_pairs, int64_t n_patches) {
    const size_t n = (size_t)n_pairs * (size_t)n_patches;
    return align_up(8 * n, 256) + align_up(4 * n, 256) + 256;
}

int geob200_fine_matching_loss_batched(const float* ref_knn_points, const float* src_knn_points, const uint8_t* ref_knn_masks,
                                       const uint8_t* src_knn_masks, const float* matching_scores, const float* transforms, int64_t n_pairs,
                                       int64_t n_patches, int64_t k, const int32_t* patch_count, double positive_radius,
                                       const float* loss_weights, float* out, int64_t out_ld, void* workspace, size_t workspace_bytes,
                                       void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "fine_matching_loss_batched: 1..65535 pairs");
    GEOB_REQUIRE(n_patches >= 0 && n_patches < (1 << 30), "fine_matching_loss_batched: negative patch count");
    GEOB_REQUIRE(k == 64 || k == 128, "fine_matching_loss_batched: k must be 64 or 128, got %lld", (long long)k);
    GEOB_REQUIRE(positive_radius > 0.0, "fine_matching_loss_batched: positive_radius must be positive");
    GEOB_REQUIRE(out_ld >= 3, "fine_matching_loss_batched: out_ld >= 3 required");
    GEOB_REQUIRE(workspace_bytes >= geob200_fine_matching_loss_batched_workspace_bytes(n_pairs, n_patches),
                 "fine_matching_loss_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    double* psum = ar.take<double>((size_t)n_pairs * n_patches);
    int* pcnt = ar.take<int>((size_t)n_pairs * n_patches);
    GEOB_REQUIRE(ar.ok(), "fine_matching_loss_batched: workspace accounting error");
    const float r2 = (float)(positive_radius * positive_radius);      // radius ** 2 in double, rounded once (torch.lt against it)
    const int P = (int)n_patches;
    float w_c = 0.f, w_f = 0.f;
    if (loss_weights != nullptr) { w_c = loss_weights[0]; w_f = loss_weights[1]; }
    int n_launch = 1;
    if (P > 0) {
        const dim3 grid((unsigned)P, (unsigned)n_pairs);
        if (k == 64)
            floss_patch_kernel<64><<<grid, 256, 0, st>>>(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, matching_scores,
                                                         transforms, P, patch_count, r2, psum, pcnt);
        else
            floss_patch_kernel<128><<<grid, 256, 0, st>>>(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, matching_scores,
                                                          transforms, P, patch_count, r2, psum, pcnt);
        n_launch += 1;
    }
    floss_finalize_kernel<<<(unsigned)n_pairs, 32, 0, st>>>(psum, pcnt, P, loss_weights != nullptr, w_c, w_f, out, (long long)out_ld);
    GEOB_CHECK_LAUNCH();
    count_launches(n_launch);
    return 0;
}

}  // extern "C"
