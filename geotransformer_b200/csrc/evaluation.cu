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
// Cloud s = blockIdx.y; clouds s < B are the ref clouds (inputs from the ref_* block at cl.start[s]), the others the src clouds (inputs
// from the src_* block, which starts at cloud B), transformed by T + 16 * (s - B).  Outputs are stacked at cl.start[s].
__global__ void __launch_bounds__(256) nc_prepare_kernel(const float* __restrict__ ref_nodes, const float* __restrict__ src_nodes,
                                                         const float* __restrict__ ref_knn_pts, const float* __restrict__ src_knn_pts,
                                                         const unsigned char* __restrict__ ref_knn_masks,
                                                         const unsigned char* __restrict__ src_knn_masks, const __grid_constant__ Segs cl,
                                                         int B, int K, const float* __restrict__ T, float* __restrict__ nodes_out,
                                                         float* __restrict__ pts_out, float* __restrict__ max_dist, int* __restrict__ n_valid) {
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.y;
    const int m = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (m >= cl.count[s]) return;
    const bool src = s >= B;
    const float* __restrict__ nodes = src ? src_nodes : ref_nodes;
    const float* __restrict__ knn_pts = src ? src_knn_pts : ref_knn_pts;
    const unsigned char* __restrict__ knn_masks = src ? src_knn_masks : ref_knn_masks;
    {
        const long long r = cl.start[s], r_in = src ? r - cl.start[B] : r;
        nodes += 3 * r_in; knn_pts += 3 * r_in * K; nodes_out += 3 * r; pts_out += 3 * r * K; max_dist += r; n_valid += r;
        if (knn_masks != nullptr) knn_masks += r_in * K;
        T = (T != nullptr && src) ? T + 16 * (s - B) : nullptr;
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
// live (may be NULL): 2 - 2 <f_i, g_j> >= 0, where the clamp passes its gradient (the backward).
__global__ void __launch_bounds__(256) closs_dist_kernel(const float* __restrict__ fr, const float* __restrict__ fs, int C,
                                                         const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                         const __grid_constant__ Segs NN, float* __restrict__ d, float* __restrict__ o,
                                                         unsigned char* __restrict__ live) {
    extern __shared__ float a[];            // [C]
    const int p = blockIdx.y, i = blockIdx.x;
    const int M = R.count[p], N = Q.count[p];
    if (i >= M) return;
    fr += ((long long)R.start[p] + i) * C;
    fs += (long long)Q.start[p] * C;
    d += NN.start[p] + (long long)i * N;
    o += NN.start[p] + (long long)i * N;
    if (live != nullptr) live += NN.start[p] + (long long)i * N;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = threadIdx.x; c < C; c += blockDim.x) a[c] = fr[c];
    __syncthreads();
    for (int j = warp; j < N; j += 8) {
        const float* b = fs + (long long)j * C;
        float x = 0.f;
        for (int c = lane; c < C; c += 32) x = fmaf(a[c], b[c], x);
        x = warp_sum(x);
        if (lane == 0) {
            const float y = __fsub_rn(2.0f, __fmul_rn(2.0f, x));
            d[j] = sqrtf(fmaxf(y, 0.0f));
            o[j] = 0.f;
            if (live != nullptr) live[j] = y >= 0.0f;
        }
    }
}

// o[i][j] = overlap of the first count[p] ground-truth rows of pair p (rows at NN.start[p]); a row whose (i, j) lies outside the
// pair's n_ref x n_src matrix is skipped (the indices come from the caller's output dict)
__global__ void __launch_bounds__(256) closs_scatter_kernel(const long long* __restrict__ gt_idx, const float* __restrict__ gt_ov,
                                                            const int* __restrict__ count, const __grid_constant__ Segs R,
                                                            const __grid_constant__ Segs Q, const __grid_constant__ Segs NN,
                                                            float* __restrict__ o) {
    const int p = blockIdx.y;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(count[p], NN.count[p]);
    if (g >= n) return;
    gt_idx += 2ll * NN.start[p]; gt_ov += NN.start[p];
    const long long i = gt_idx[2ll * g], j = gt_idx[2ll * g + 1];
    if ((unsigned long long)i >= (unsigned long long)R.count[p] || (unsigned long long)j >= (unsigned long long)Q.count[p]) return;
    o[NN.start[p] + i * Q.count[p] + j] = gt_ov[g];
}

struct CircleParams {
    float pos_margin, neg_margin, pos_optimal, neg_optimal, log_scale, pos_overlap;
};

// circle_loss.py:56-76 for one entry: positive / negative flags, the detached weights wp / wn and the logits lp / ln
__device__ __forceinline__ void circle_logits(const CircleParams& cp, float dv, float ov, float& lp, float& ln, int& pos, int& neg, float& wp,
                                              float& wn) {
    pos = ov > cp.pos_overlap;
    neg = ov == 0.f;
    wp = pos ? __fmul_rn(fmaxf(__fsub_rn(dv, cp.pos_optimal), 0.f), sqrtf(ov)) : 0.f;
    wn = neg ? fmaxf(__fsub_rn(cp.neg_optimal, dv), 0.f) : 0.f;
    lp = __fmul_rn(__fmul_rn(cp.log_scale, __fsub_rn(dv, cp.pos_margin)), wp);
    ln = __fmul_rn(__fmul_rn(cp.log_scale, __fsub_rn(cp.neg_margin, dv)), wn);
}

// one CTA per row (blockIdx.z = 0: ref superpoint i over all j) or column (z = 1: src superpoint j over all i) of pair blockIdx.y:
// both logsumexps (max subtracted first), loss = softplus(Lp + Ln) / log_scale and kept = (has a positive and a negative).
// Weight-0 entries stay in the sums (exp(0) = 1), as in the reference.  Results at the row's / column's cloud offset.
// lse_r / lse_c (may be NULL): the two logsumexps of the line (the backward).
__global__ void __launch_bounds__(256) closs_lse_kernel(const float* __restrict__ d, const float* __restrict__ o,
                                                        const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                        const __grid_constant__ Segs NN, CircleParams cp, float* __restrict__ ell_r,
                                                        unsigned char* __restrict__ kept_r, float* __restrict__ ell_c,
                                                        unsigned char* __restrict__ kept_c, float2* __restrict__ lse_r,
                                                        float2* __restrict__ lse_c) {
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
        float wp, wn;
        circle_logits(cp, d[base + e * step], o[base + e * step], lp, ln, pos, neg, wp, wn);
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
        if (lse_r != nullptr) (col ? lse_c : lse_r)[r] = make_float2(mp + logf(sp), mn + logf(sn));
    }
}

// Backward of c_loss.  Per pair: g = upstream gradient of c_loss (grad[p * gld + 1] + w_c * grad[p * gld] given weights); the mean
// over the kept rows / columns turns it into scale[2p] = (g / 2) / #kept rows, scale[2p + 1] = (g / 2) / #kept columns.
__global__ void __launch_bounds__(32) closs_grad_scale_kernel(const unsigned char* __restrict__ kept_r, const unsigned char* __restrict__ kept_c,
                                                              const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                              const float* __restrict__ grad, long long gld, int with_w, float w_c,
                                                              float* __restrict__ scale) {
    const int p = blockIdx.x, lane = threadIdx.x;
    const float g = with_w ? grad[p * gld + 1] + w_c * grad[p * gld] : grad[p * gld + 1];
    for (int side = 0; side < 2; ++side) {
        const unsigned char* kept = side ? kept_c : kept_r;
        const int s0 = side ? Q.start[p] : R.start[p], n = side ? Q.count[p] : R.count[p];
        int k = 0;
        for (int i = lane; i < n; i += 32) k += kept[s0 + i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
        if (lane == 0) scale[2 * p + side] = (g / 2.0f) / (float)k;
    }
}

// torch softplus backward (beta 1, threshold 20) of l = softplus(x) / log_scale, for a line whose loss enters the mean with `scale`
__device__ __forceinline__ float closs_line_grad(float2 lse, bool kept, float scale, float log_scale) {
    if (!kept) return 0.f;
    const float x = lse.x + lse.y, gl = scale / log_scale;
    if (x > 20.f) return gl;
    const float z = expf(x);
    return gl * z / (z + 1.f);
}

// dc_loss / d<f_i, g_j> for every entry (i, j) of pair p, written over o: the logsumexp softmaxes of the entry's row and column, the
// detached weights, then sqrt (grad / (2 d)) and the clamp (zero where 2 - 2 <f, g> < 0) in torch's order -- so an entry at d = 0
// gives inf or NaN exactly where torch autograd does.
__global__ void __launch_bounds__(256) closs_grad_kernel(const float* __restrict__ d, float* __restrict__ o, const unsigned char* __restrict__ live,
                                                         const float2* __restrict__ lse_r, const float2* __restrict__ lse_c,
                                                         const unsigned char* __restrict__ kept_r, const unsigned char* __restrict__ kept_c,
                                                         const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                         const __grid_constant__ Segs NN, CircleParams cp, const float* __restrict__ scale) {
    const int p = blockIdx.y;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= NN.count[p]) return;
    const int N = Q.count[p];
    const int i = (int)(t / N), j = (int)(t % N);
    const long long e = NN.start[p] + t;
    const float dv = d[e];
    float lp, ln, wp, wn;
    int pos, neg;
    circle_logits(cp, dv, o[e], lp, ln, pos, neg, wp, wn);
    const float2 lr = lse_r[R.start[p] + i], lc = lse_c[Q.start[p] + j];
    const float gr = closs_line_grad(lr, kept_r[R.start[p] + i], scale[2 * p], cp.log_scale);
    const float gc = closs_line_grad(lc, kept_c[Q.start[p] + j], scale[2 * p + 1], cp.log_scale);
    const float glp = gr * expf(lp - lr.x) + gc * expf(lp - lc.x);
    const float gln = gr * expf(ln - lr.y) + gc * expf(ln - lc.y);
    const float gd = (glp * wp) * cp.log_scale - (gln * wn) * cp.log_scale;
    const float gsq = live[e] ? gd / (2.0f * dv) : 0.f;
    o[e] = -gsq * 2.0f;
}

// grad_ref[i] = sum_j G[i][j] fs[j] (side 0, blockIdx.z) and grad_src[j] = sum_i G[i][j] fr[i] (side 1), summed in index order
__global__ void __launch_bounds__(128) closs_feat_grad_kernel(const float* __restrict__ G, const float* __restrict__ fr,
                                                              const float* __restrict__ fs, int C, const __grid_constant__ Segs R,
                                                              const __grid_constant__ Segs Q, const __grid_constant__ Segs NN,
                                                              float* __restrict__ grad_ref, float* __restrict__ grad_src) {
    const int p = blockIdx.y, side = blockIdx.z, line = blockIdx.x;
    const int M = R.count[p], N = Q.count[p];
    if (line >= (side ? N : M)) return;
    G += NN.start[p];
    const float* other = side ? fr + (long long)R.start[p] * C : fs + (long long)Q.start[p] * C;
    float* out = side ? grad_src + ((long long)Q.start[p] + line) * C : grad_ref + ((long long)R.start[p] + line) * C;
    const int n = side ? M : N;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < n; ++k) s += G[side ? (long long)k * N + line : (long long)line * N + k] * other[(long long)k * C + c];
        out[c] = s;
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
// MODE 0: the values above; 1: #labels only (scores unread); 2: the backward -- every entry of the block gets -g_p / n_p on a label
// and 0 elsewhere, with n_p = the pair's #labels from a MODE 1 pass in pcnt and g_p the upstream gradient of f_loss (grad[p * gld + 2]
// + w_f * grad[p * gld] given weights) -- written to scores.
template <int K, int MODE>
__global__ void __launch_bounds__(256) floss_patch_kernel(const float* __restrict__ ref_pts, const float* __restrict__ src_pts,
                                                          const unsigned char* __restrict__ ref_masks,
                                                          const unsigned char* __restrict__ src_masks, float* __restrict__ scores,
                                                          const float* __restrict__ T, int P, const int* __restrict__ count, float r2,
                                                          double* __restrict__ psum, int* __restrict__ pcnt, const float* __restrict__ grad,
                                                          long long gld, int with_w, float w_f) {
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
    float* S = scores + patch * (K + 1) * (K + 1);
    double s = 0.0;
    int n = 0;
    auto hit = [&](int i, int j) {
        const float4 a = rp[i], b = sp[j];
        return a.w >= 0.f && b.w >= 0.f && sqd_mm(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w) < r2;
    };
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
        const int i = e / K, j = e % K;
        if (hit(i, j)) {
            rhit[i] = 1;
            shit[j] = 1;
            if (MODE == 0) s += S[i * (K + 1) + j];
            ++n;
        }
    }
    __syncthreads();
    if constexpr (MODE == 2) {
        int np = 0;
        for (int k = threadIdx.x; k < P; k += blockDim.x) np += pcnt[(long long)p * P + k];
        np = block_reduce_256(np, [](int x, int y) { return x + y; }, redi);
        const float g = with_w ? grad[p * gld + 2] + w_f * grad[p * gld] : grad[p * gld + 2];
        const float val = np > 0 ? -g / (float)np : 0.f;
        for (int e = threadIdx.x; e < (K + 1) * (K + 1); e += blockDim.x) {
            const int i = e / (K + 1), j = e % (K + 1);
            bool lab;
            if (i < K && j < K) lab = hit(i, j);
            else if (i < K && j == K) lab = rp[i].w >= 0.f && !rhit[i];
            else if (i == K && j < K) lab = sp[j].w >= 0.f && !shit[j];
            else lab = false;
            S[e] = lab ? val : 0.f;
        }
    } else {
        for (int i = threadIdx.x; i < K; i += blockDim.x) {
            if (rp[i].w >= 0.f && !rhit[i]) { if (MODE == 0) s += S[i * (K + 1) + K]; ++n; }
            if (sp[i].w >= 0.f && !shit[i]) { if (MODE == 0) s += S[K * (K + 1) + i]; ++n; }
        }
        if (MODE == 0) s = block_reduce_256(s, [](double x, double y) { return x + y; }, redd);
        n = block_reduce_256(n, [](int x, int y) { return x + y; }, redi);
        if (threadIdx.x == 0) {
            if (MODE == 0) psum[patch] = s;
            pcnt[patch] = n;
        }
    }
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

size_t geob200_node_correspondences_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t k) {
    const size_t r = (size_t)n_rows;
    return align_up(12 * r, 256) + align_up(12 * r * (size_t)k, 256) + 2 * align_up(4 * r, 256) + align_up(4 * (size_t)n_products, 256) + 256;
}

int geob200_node_correspondences_batched(const float* ref_nodes, const float* src_nodes, const float* ref_knn_points,
                                         const float* src_knn_points, const uint8_t* ref_masks, const uint8_t* src_masks,
                                         const uint8_t* ref_knn_masks, const uint8_t* src_knn_masks, int64_t n_pairs, const int64_t* cloud_nodes,
                                         int64_t k, const float* transforms, float pos_radius, int64_t* corr_indices, float* corr_overlaps,
                                         int32_t* count, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "node_correspondences_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(k > 0 && k <= 1024, "node_correspondences: bad shape");
    const int B = (int)n_pairs;
    // cl: all 2B clouds stacked (the workspace rows); R / Q: the ref / src clouds in the row spaces of the ref_* / src_* inputs
    Segs cl, Q, NN;
    if (segs_from_counts(&cl, 2 * n_pairs, cloud_nodes) || segs_from_counts(&Q, n_pairs, cloud_nodes + n_pairs)) return -1;
    const Segs R = segs_range(cl, 0, B);
    const int64_t ref_rows = cl.start[B], rows = (int64_t)cl.start[2 * B - 1] + cl.count[2 * B - 1];
    GEOB_REQUIRE(ref_rows > 0 && rows > ref_rows, "node_correspondences: bad shape");
    if (segs_products(&NN, R, Q)) return -1;
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
        ref_nodes, src_nodes, ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, cl, B, (int)k, transforms, cn, cp, cmax, cnv);
    const size_t smem = (size_t)k * (2 * sizeof(float4) + 2 * sizeof(int));
    if (R.max > 0)
        nc_overlap_kernel<<<dim3((unsigned)R.max, B), 256, smem, st>>>(cn, cn + 3 * ref_rows, cp, cp + 3 * ref_rows * k, ref_knn_masks,
                                                                      src_knn_masks, ref_masks, src_masks, cmax, cmax + ref_rows, cnv,
                                                                      cnv + ref_rows, R, Q, NN, (int)k, pos_radius, overlap);
    nc_compact_kernel<<<B, 1024, 0, st>>>(overlap, R, Q, NN, (long long*)corr_indices, corr_overlaps, count);
    GEOB_CHECK_LAUNCH();
    count_launches(3);
    return 0;
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
        closs_dist_kernel<<<dim3((unsigned)R.max, B), 256, channels * sizeof(float), st>>>(ref_feats, src_feats, (int)channels, R, Q, NN, d, o,
                                                                                           nullptr);
        closs_scatter_kernel<<<dim3((unsigned)((NN.max + 255) / 256), B), 256, 0, st>>>((const long long*)gt_node_corr_indices,
                                                                                        gt_node_corr_overlaps, gt_count, R, Q, NN, o);
        n_launch += 2;
    }
    if (R.max > 0 || Q.max > 0) {
        closs_lse_kernel<<<dim3((unsigned)(R.max > Q.max ? R.max : Q.max), B, 2), 256, 0, st>>>(d, o, R, Q, NN, cp, ell, kept, ell_c, kept_c,
                                                                                                nullptr, nullptr);
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
            floss_patch_kernel<64, 0><<<grid, 256, 0, st>>>(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks,
                                                            const_cast<float*>(matching_scores), transforms, P, patch_count, r2, psum, pcnt,
                                                            nullptr, 0, 0, 0.f);
        else
            floss_patch_kernel<128, 0><<<grid, 256, 0, st>>>(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks,
                                                             const_cast<float*>(matching_scores), transforms, P, patch_count, r2, psum, pcnt,
                                                             nullptr, 0, 0, 0.f);
        n_launch += 1;
    }
    floss_finalize_kernel<<<(unsigned)n_pairs, 32, 0, st>>>(psum, pcnt, P, loss_weights != nullptr, w_c, w_f, out, (long long)out_ld);
    GEOB_CHECK_LAUNCH();
    count_launches(n_launch);
    return 0;
}

size_t geob200_coarse_matching_loss_backward_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t n_pairs) {
    const size_t r = (size_t)n_rows, nn = (size_t)n_products;
    return geob200_coarse_matching_loss_batched_workspace_bytes(n_rows, n_products) + align_up(nn, 256) + align_up(8 * r, 256) +
           align_up(8 * (size_t)n_pairs, 256) + 1024;
}

int geob200_coarse_matching_loss_backward_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs,
                                                  const int64_t* cloud_nodes, const int64_t* gt_node_corr_indices,
                                                  const float* gt_node_corr_overlaps, const int32_t* gt_count, float positive_margin,
                                                  float negative_margin, float positive_optimal, float negative_optimal, float log_scale,
                                                  float positive_overlap, const float* grad_rows, int64_t grad_ld, const float* loss_weights,
                                                  float* grad_ref_feats, float* grad_src_feats, void* workspace, size_t workspace_bytes,
                                                  void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "coarse_matching_loss_backward_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(channels > 0 && channels <= 8192, "coarse_matching_loss_backward_batched: 1..8192 channels");
    GEOB_REQUIRE(log_scale > 0.f, "coarse_matching_loss_backward_batched: log_scale must be positive");
    GEOB_REQUIRE(grad_ld >= 3, "coarse_matching_loss_backward_batched: grad_ld >= 3 required");
    GEOB_REQUIRE(gt_count != nullptr && grad_rows != nullptr && grad_ref_feats != nullptr && grad_src_feats != nullptr,
                 "coarse_matching_loss_backward_batched: null pointer");
    for (int64_t c = 0; c < 2 * n_pairs; ++c) GEOB_REQUIRE(cloud_nodes[c] >= 0, "coarse_matching_loss_backward_batched: negative node count");
    const int B = (int)n_pairs;
    Segs R, Q, NN;
    if (segs_from_counts(&R, B, cloud_nodes) || segs_from_counts(&Q, B, cloud_nodes + B) || segs_products(&NN, R, Q)) return -1;
    const int64_t n_ref = (int64_t)R.start[B - 1] + R.count[B - 1];
    const int64_t rows = n_ref + Q.start[B - 1] + Q.count[B - 1];
    const int64_t nn = (int64_t)NN.start[B - 1] + NN.count[B - 1];
    GEOB_REQUIRE(workspace_bytes >= geob200_coarse_matching_loss_backward_batched_workspace_bytes(rows, nn, n_pairs),
                 "coarse_matching_loss_backward_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    float* d = ar.take<float>(nn);
    float* o = ar.take<float>(nn);                           // overlaps, then dc_loss / d<f, g>
    float* ell = ar.take<float>(rows);
    unsigned char* kept = ar.take<unsigned char>(rows);
    unsigned char* live = ar.take<unsigned char>(nn);
    float2* lse = ar.take<float2>(rows);
    float* scale = ar.take<float>(2 * (size_t)B);
    GEOB_REQUIRE(ar.ok(), "coarse_matching_loss_backward_batched: workspace accounting error");
    const CircleParams cp{positive_margin, negative_margin, positive_optimal, negative_optimal, log_scale, positive_overlap};
    const float w_c = loss_weights != nullptr ? loss_weights[0] : 0.f;
    int n_launch = 1;
    if (R.max > 0 && Q.max > 0) {
        closs_dist_kernel<<<dim3((unsigned)R.max, B), 256, channels * sizeof(float), st>>>(ref_feats, src_feats, (int)channels, R, Q, NN, d, o,
                                                                                           live);
        closs_scatter_kernel<<<dim3((unsigned)((NN.max + 255) / 256), B), 256, 0, st>>>((const long long*)gt_node_corr_indices,
                                                                                        gt_node_corr_overlaps, gt_count, R, Q, NN, o);
        closs_lse_kernel<<<dim3((unsigned)(R.max > Q.max ? R.max : Q.max), B, 2), 256, 0, st>>>(d, o, R, Q, NN, cp, ell, kept, ell + n_ref,
                                                                                                kept + n_ref, lse, lse + n_ref);
        closs_grad_scale_kernel<<<B, 32, 0, st>>>(kept, kept + n_ref, R, Q, grad_rows, (long long)grad_ld, loss_weights != nullptr, w_c,
                                                  scale);
        closs_grad_kernel<<<dim3((unsigned)((NN.max + 255) / 256), B), 256, 0, st>>>(d, o, live, lse, lse + n_ref, kept, kept + n_ref, R,
                                                                                      Q, NN, cp, scale);
        n_launch += 5;
    }
    // every feature row is written (zeros for a cloud whose partner is empty)
    closs_feat_grad_kernel<<<dim3((unsigned)(R.max > Q.max ? R.max : Q.max) + (R.max == 0 && Q.max == 0), B, 2), 128, 0, st>>>(
        o, ref_feats, src_feats, (int)channels, R, Q, NN, grad_ref_feats, grad_src_feats);
    GEOB_CHECK_LAUNCH();
    count_launches(n_launch);
    return 0;
}

size_t geob200_fine_matching_loss_backward_batched_workspace_bytes(int64_t n_pairs, int64_t n_patches) {
    return align_up(4 * (size_t)n_pairs * (size_t)n_patches, 256) + 256;
}

int geob200_fine_matching_loss_backward_batched(const float* ref_knn_points, const float* src_knn_points, const uint8_t* ref_knn_masks,
                                                const uint8_t* src_knn_masks, const float* transforms, int64_t n_pairs, int64_t n_patches,
                                                int64_t k, const int32_t* patch_count, double positive_radius, const float* grad_rows,
                                                int64_t grad_ld, const float* loss_weights, float* grad_scores, void* workspace,
                                                size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= 65535, "fine_matching_loss_backward_batched: 1..65535 pairs");
    GEOB_REQUIRE(n_patches >= 0 && n_patches < (1 << 30), "fine_matching_loss_backward_batched: negative patch count");
    GEOB_REQUIRE(k == 64 || k == 128, "fine_matching_loss_backward_batched: k must be 64 or 128, got %lld", (long long)k);
    GEOB_REQUIRE(positive_radius > 0.0, "fine_matching_loss_backward_batched: positive_radius must be positive");
    GEOB_REQUIRE(grad_ld >= 3, "fine_matching_loss_backward_batched: grad_ld >= 3 required");
    GEOB_REQUIRE(grad_rows != nullptr && (n_patches == 0 || grad_scores != nullptr), "fine_matching_loss_backward_batched: null pointer");
    GEOB_REQUIRE(workspace_bytes >= geob200_fine_matching_loss_backward_batched_workspace_bytes(n_pairs, n_patches),
                 "fine_matching_loss_backward_batched: workspace too small");
    if (n_patches == 0) return 0;
    Arena ar(workspace, workspace_bytes);
    int* pcnt = ar.take<int>((size_t)n_pairs * n_patches);
    GEOB_REQUIRE(ar.ok(), "fine_matching_loss_backward_batched: workspace accounting error");
    const float r2 = (float)(positive_radius * positive_radius);
    const int P = (int)n_patches;
    const float w_f = loss_weights != nullptr ? loss_weights[1] : 0.f;
    const int with_w = loss_weights != nullptr;
    const dim3 grid((unsigned)P, (unsigned)n_pairs);
#define LAUNCH_FLB(KV, MODE)                                                                                                          \
    floss_patch_kernel<KV, MODE><<<grid, 256, 0, st>>>(ref_knn_points, src_knn_points, ref_knn_masks, src_knn_masks, grad_scores,      \
                                                       transforms, P, patch_count, r2, nullptr, pcnt, grad_rows, (long long)grad_ld,   \
                                                       with_w, w_f)
    if (k == 64) { LAUNCH_FLB(64, 1); LAUNCH_FLB(64, 2); }
    else { LAUNCH_FLB(128, 1); LAUNCH_FLB(128, 2); }
#undef LAUNCH_FLB
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

}  // extern "C"

// ---- RPMNet's ModelNet metrics (modified Chamfer distance, anisotropic errors) --------------------------------------------------
//
// Reference: geotransformer/utils/registration.py:69-130 (compute_rotation_mse_and_mae, compute_translation_mse_and_mae,
// compute_modified_chamfer_distance) and modules/registration/metrics.py:8-161.  The contract is in DESIGN.md section 8a:
//   cd_pq = mean_i |fp32(est src_i) - raw_nn|, cd_qp = mean_j |ref_j - fp32((est gt^-1) raw)_nn|, exact nearest neighbours with fp64
//   distances (feature_nn_launch, C = 3); transforms composed and applied in fp64 and rounded to fp32 once; per-pair sums in a fixed
//   order.  r_mse / r_mae: scipy's from_matrix (polar factor unless the Gram matrix is within isclose(atol=1e-12) of I, Shepperd's
//   quaternion) and as_euler('xyz', degrees=True) with its gimbal rule, differences not wrapped; t_mse / t_mae in fp32 as numpy.
#include "feature_match.cuh"
#include "kabsch.cuh"

namespace geob200 {

constexpr int RP_MAX_PAIRS = GEOB_MAX_CLOUDS / 2;
constexpr int RP_THREADS = 256;

struct RpLaunch {
    int n;
    int cap_q, cap_s;                          // rows per pair of the query (src, ref) and support (raw) buffers
    long long raw0[RP_MAX_PAIRS], ref0[RP_MAX_PAIRS], src0[RP_MAX_PAIRS];
    int n_raw[RP_MAX_PAIRS], n_ref[RP_MAX_PAIRS], n_src[RP_MAX_PAIRS];
};

__device__ __forceinline__ double det3(const double* m) {
    return __dsub_rn(__dadd_rn(__dmul_rn(m[0], __dsub_rn(__dmul_rn(m[4], m[8]), __dmul_rn(m[5], m[7]))),
                               __dmul_rn(m[2], __dsub_rn(__dmul_rn(m[3], m[7]), __dmul_rn(m[4], m[6])))),
                     __dmul_rn(m[1], __dsub_rn(__dmul_rn(m[3], m[8]), __dmul_rn(m[5], m[6]))));
}

// scipy's Rotation.from_matrix(M).as_euler('xyz') in radians, M with det > 0 (fp32 values widened to fp64, as from_matrix does)
__device__ void rp_euler_xyz(const double (&Min)[9], double (&e)[3]) {
    double M[9];
    for (int i = 0; i < 9; ++i) M[i] = Min[i];
    bool orthogonal = true;                    // isclose(M M^T, I, rtol=1e-5, atol=1e-12) everywhere
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const double g = __dadd_rn(__dadd_rn(__dmul_rn(M[3 * i], M[3 * j]), __dmul_rn(M[3 * i + 1], M[3 * j + 1])),
                                       __dmul_rn(M[3 * i + 2], M[3 * j + 2]));
            const double want = i == j ? 1.0 : 0.0;
            if (!(fabs(g - want) <= 1e-12 + 1e-5 * want)) orthogonal = false;
        }
    if (!orthogonal) {                         // the polar factor U V^T of M = U S V^T: kabsch_rotation(M^T) (det M > 0: no flip)
        double Mt[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) Mt[3 * i + j] = M[3 * j + i];
        kabsch_rotation(Mt, M);
    }
    // Shepperd: argmax (first on ties) of [m00, m11, m22, trace]; quaternion (x, y, z, w), normalised
    const double tr = __dadd_rn(__dadd_rn(M[0], M[4]), M[8]);
    const double dec[4] = {M[0], M[4], M[8], tr};
    int c = 0;
    for (int k = 1; k < 4; ++k)
        if (dec[k] > dec[c]) c = k;
    double q[4];
    if (c == 3) {
        q[0] = __dsub_rn(M[7], M[5]); q[1] = __dsub_rn(M[2], M[6]); q[2] = __dsub_rn(M[3], M[1]); q[3] = __dadd_rn(1.0, tr);
    } else {
        const int i = c, j = (i + 1) % 3, k = (j + 1) % 3;
        q[i] = __dadd_rn(__dsub_rn(1.0, tr), __dmul_rn(2.0, M[4 * i]));
        q[j] = __dadd_rn(M[3 * j + i], M[3 * i + j]);
        q[k] = __dadd_rn(M[3 * k + i], M[3 * i + k]);
        q[3] = __dsub_rn(M[3 * k + j], M[3 * j + k]);
    }
    const double nq = __dsqrt_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])),
                                           __dmul_rn(q[3], q[3])));
    for (int k = 0; k < 4; ++k) q[k] = __ddiv_rn(q[k], nq);
    // as_euler, extrinsic 'xyz' (i, j, k = 0, 1, 2; sign = 1)
    const double a = __dsub_rn(q[3], q[1]), b = __dadd_rn(q[0], q[2]), cc = __dadd_rn(q[1], q[3]), d = __dsub_rn(q[2], q[0]);
    const double second = __dmul_rn(2.0, atan2(hypot(cc, d), hypot(a, b)));
    const double half_sum = atan2(b, a), half_diff = atan2(d, cc);
    if (fabs(second) <= 1e-7) {                // gimbal lock: third angle 0
        e[0] = __dmul_rn(2.0, half_sum); e[2] = 0.0;
    } else if (fabs(__dsub_rn(second, M_PI)) <= 1e-7) {
        e[0] = -__dmul_rn(2.0, half_diff); e[2] = 0.0;
    } else {
        e[0] = __dsub_rn(half_sum, half_diff); e[2] = __dadd_rn(half_sum, half_diff);
    }
    e[1] = __dsub_rn(second, M_PI_2);
    for (int k = 0; k < 3; ++k) {
        if (e[k] < -M_PI) e[k] = __dadd_rn(e[k], 2.0 * M_PI);
        else if (e[k] > M_PI) e[k] = __dsub_rn(e[k], 2.0 * M_PI);
    }
}

// One thread per pair: the status (det <= 0 of gt or est), the anisotropic errors, and the two transforms the points kernel applies
// (est, and est gt^-1 with gt^-1 = [A^-1 | -A^-1 t] by the adjugate), 12 doubles each, in xf.
__global__ void __launch_bounds__(32) rp_pair_kernel(int n, const float* __restrict__ gt, const float* __restrict__ est,
                                                     double* __restrict__ xf, double* __restrict__ out) {
    const int p = threadIdx.x;
    if (p >= n) return;
    const float* G = gt + 16 * p;
    const float* E = est + 16 * p;
    double Rg[9], Re[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { Rg[3 * i + j] = (double)G[4 * i + j]; Re[3 * i + j] = (double)E[4 * i + j]; }
    double* o = out + GEOB200_RPMNET_COLUMNS * p;
    const double dg = det3(Rg), de = det3(Re);
    o[7] = !(dg > 0.0) ? GEOB200_RPMNET_GT_DET : !(de > 0.0) ? GEOB200_RPMNET_EST_DET : 0;
    if (o[7] == 0.0) {
        double eg[3], ee[3];
        rp_euler_xyz(Rg, eg);
        rp_euler_xyz(Re, ee);
        const double deg = 180.0 / M_PI;       // np.rad2deg
        double s2 = 0.0, s1 = 0.0;
        for (int k = 0; k < 3; ++k) {
            const double t = __dsub_rn(__dmul_rn(eg[k], deg), __dmul_rn(ee[k], deg));
            s2 = __dadd_rn(s2, __dmul_rn(t, t));
            s1 = __dadd_rn(s1, fabs(t));
        }
        o[3] = __ddiv_rn(s2, 3.0);
        o[4] = __ddiv_rn(s1, 3.0);
    } else {
        o[3] = o[4] = __longlong_as_double(0x7ff8000000000000ll);
    }
    float f2 = 0.0f, f1 = 0.0f;                // fp32 translation errors, as numpy's float32 mean of three
    for (int i = 0; i < 3; ++i) {
        const float t = __fsub_rn(G[4 * i + 3], E[4 * i + 3]);
        f2 = __fadd_rn(f2, __fmul_rn(t, t));
        f1 = __fadd_rn(f1, fabsf(t));
    }
    o[5] = (double)__fdiv_rn(f2, 3.0f);
    o[6] = (double)__fdiv_rn(f1, 3.0f);
    // est, then est gt^-1
    double* x = xf + 24 * p;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) x[4 * i + j] = Re[3 * i + j];
        x[4 * i + 3] = (double)E[4 * i + 3];
    }
    double Ai[9];
    const double id = 1.0 / dg;
    Ai[0] = (Rg[4] * Rg[8] - Rg[5] * Rg[7]) * id; Ai[1] = (Rg[2] * Rg[7] - Rg[1] * Rg[8]) * id; Ai[2] = (Rg[1] * Rg[5] - Rg[2] * Rg[4]) * id;
    Ai[3] = (Rg[5] * Rg[6] - Rg[3] * Rg[8]) * id; Ai[4] = (Rg[0] * Rg[8] - Rg[2] * Rg[6]) * id; Ai[5] = (Rg[2] * Rg[3] - Rg[0] * Rg[5]) * id;
    Ai[6] = (Rg[3] * Rg[7] - Rg[4] * Rg[6]) * id; Ai[7] = (Rg[1] * Rg[6] - Rg[0] * Rg[7]) * id; Ai[8] = (Rg[0] * Rg[4] - Rg[1] * Rg[3]) * id;
    double ti[3];
    for (int i = 0; i < 3; ++i) ti[i] = -(Ai[3 * i] * G[3] + Ai[3 * i + 1] * G[7] + Ai[3 * i + 2] * G[11]);
    double* y = x + 12;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) y[4 * i + j] = Re[3 * i] * Ai[j] + Re[3 * i + 1] * Ai[3 + j] + Re[3 * i + 2] * Ai[6 + j];
        y[4 * i + 3] = Re[3 * i] * ti[0] + Re[3 * i + 1] * ti[1] + Re[3 * i + 2] * ti[2] + x[4 * i + 3];
    }
}

__device__ __forceinline__ void rp_apply(const double* T, const float* p, float* q) {
    const double x = p[0], y = p[1], z = p[2];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        q[i] = __double2float_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * i], x), __dmul_rn(T[4 * i + 1], y)), __dmul_rn(T[4 * i + 2], z)),
                                           T[4 * i + 3]));
}

// Grid (ceil(max rows / RP_THREADS), n): the padded nearest-neighbour inputs of pair p.  Queries: slot p = est src, slot n + p = ref;
// supports: slot p = raw, slot n + p = (est gt^-1) raw.
__global__ void __launch_bounds__(RP_THREADS) rp_points_kernel(const __grid_constant__ RpLaunch L, const float* __restrict__ raw,
                                                               const float* __restrict__ ref, const float* __restrict__ src,
                                                               const double* __restrict__ xf, float* __restrict__ Q, float* __restrict__ S,
                                                               int32_t* __restrict__ nq, int32_t* __restrict__ ns) {
    const int p = blockIdx.y, r = blockIdx.x * RP_THREADS + threadIdx.x, n = L.n;
    const double* x = xf + 24 * p;
    if (r == 0) { nq[p] = L.n_src[p]; nq[n + p] = L.n_ref[p]; ns[p] = L.n_raw[p]; ns[n + p] = L.n_raw[p]; }
    if (r < L.n_src[p]) rp_apply(x, src + 3 * (L.src0[p] + r), Q + 3 * ((long long)p * L.cap_q + r));
    if (r < L.n_ref[p]) {
        const float* a = ref + 3 * (L.ref0[p] + r);
        float* b = Q + 3 * ((long long)(n + p) * L.cap_q + r);
        b[0] = a[0]; b[1] = a[1]; b[2] = a[2];
    }
    if (r < L.n_raw[p]) {
        const float* a = raw + 3 * (L.raw0[p] + r);
        float* b = S + 3 * ((long long)p * L.cap_s + r);
        b[0] = a[0]; b[1] = a[1]; b[2] = a[2];
        rp_apply(x + 12, a, S + 3 * ((long long)(n + p) * L.cap_s + r));
    }
}

// One CTA per pair: the two means of the nearest-neighbour distances, each summed per thread in row order and then by a fixed tree,
// so the bits do not depend on the batch.
__global__ void __launch_bounds__(RP_THREADS) rp_reduce_kernel(int n, int cap_q, const int32_t* __restrict__ nq, const double* __restrict__ dist,
                                                               double* __restrict__ out) {
    __shared__ double part[RP_THREADS];
    const int p = blockIdx.x, tid = threadIdx.x;
    double mean[2];
    for (int dir = 0; dir < 2; ++dir) {
        const int slot = dir * n + p, rows = nq[slot];
        const double* d = dist + (long long)slot * cap_q;
        double s = 0.0;
        for (int r = tid; r < rows; r += RP_THREADS) s = __dadd_rn(s, d[r]);
        part[tid] = s;
        __syncthreads();
        for (int h = RP_THREADS / 2; h > 0; h >>= 1) {
            if (tid < h) part[tid] = __dadd_rn(part[tid], part[tid + h]);
            __syncthreads();
        }
        mean[dir] = __ddiv_rn(part[0], (double)rows);
        __syncthreads();
    }
    if (tid == 0) {
        double* o = out + GEOB200_RPMNET_COLUMNS * p;
        o[0] = __dadd_rn(mean[0], mean[1]);
        o[1] = mean[0];
        o[2] = mean[1];
    }
}

static size_t rp_workspace(int64_t n_pairs, int64_t cap_q, int64_t cap_s) {
    const size_t B = (size_t)(n_pairs > 0 ? n_pairs : 0), q = (size_t)(cap_q > 0 ? cap_q : 0), s = (size_t)(cap_s > 0 ? cap_s : 0);
    return align_up(24 * 8 * B, 256) + align_up(2 * B * q * 12, 256) + align_up(2 * B * s * 12, 256) + 2 * align_up(8 * B, 256) +
           align_up(2 * B * q * 8, 256) + align_up(2 * B * q * 8, 256) + feature_nn_workspace(2 * (int64_t)B, q, s) + 256;
}

}  // namespace geob200

extern "C" {

size_t geob200_rpmnet_metrics_batched_workspace_bytes(int64_t n_pairs, int64_t cap_query, int64_t cap_raw) {
    return rp_workspace(n_pairs, cap_query, cap_raw);
}

int geob200_rpmnet_metrics_batched(const float* raw, const int64_t* raw_lengths_h, const float* ref, const int64_t* ref_lengths_h,
                                   const float* src, const int64_t* src_lengths_h, int64_t n_pairs, const float* gt_transforms,
                                   const float* est_transforms, double* out, void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= RP_MAX_PAIRS, "rpmnet_metrics_batched: 1..%d pairs", RP_MAX_PAIRS);
    GEOB_REQUIRE(raw_lengths_h != nullptr && ref_lengths_h != nullptr && src_lengths_h != nullptr, "rpmnet_metrics_batched: null lengths");
    GEOB_REQUIRE(raw != nullptr && ref != nullptr && src != nullptr && gt_transforms != nullptr && est_transforms != nullptr && out != nullptr,
                 "rpmnet_metrics_batched: null pointer");
    RpLaunch L{};
    L.n = (int)n_pairs;
    long long r0 = 0, f0 = 0, s0 = 0;
    for (int p = 0; p < L.n; ++p) {
        GEOB_REQUIRE(raw_lengths_h[p] > 0 && ref_lengths_h[p] > 0 && src_lengths_h[p] > 0 && raw_lengths_h[p] < (1 << 28) &&
                         ref_lengths_h[p] < (1 << 28) && src_lengths_h[p] < (1 << 28),
                     "rpmnet_metrics_batched: pair %d needs 1..2^28-1 raw, ref and src points (got %lld, %lld, %lld)", p,
                     (long long)raw_lengths_h[p], (long long)ref_lengths_h[p], (long long)src_lengths_h[p]);
        L.raw0[p] = r0; L.ref0[p] = f0; L.src0[p] = s0;
        L.n_raw[p] = (int)raw_lengths_h[p]; L.n_ref[p] = (int)ref_lengths_h[p]; L.n_src[p] = (int)src_lengths_h[p];
        r0 += raw_lengths_h[p]; f0 += ref_lengths_h[p]; s0 += src_lengths_h[p];
        L.cap_s = L.n_raw[p] > L.cap_s ? L.n_raw[p] : L.cap_s;
        L.cap_q = L.n_ref[p] > L.cap_q ? L.n_ref[p] : L.cap_q;
        L.cap_q = L.n_src[p] > L.cap_q ? L.n_src[p] : L.cap_q;
    }
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= rp_workspace(n_pairs, L.cap_q, L.cap_s),
                 "rpmnet_metrics_batched: workspace too small");
    const int B = L.n;
    Arena ar(workspace, workspace_bytes);
    double* xf = ar.take<double>(24 * (size_t)B);
    float* Q = ar.take<float>(2 * (size_t)B * L.cap_q * 3);
    float* S = ar.take<float>(2 * (size_t)B * L.cap_s * 3);
    int32_t* nq = ar.take<int32_t>(2 * (size_t)B);
    int32_t* ns = ar.take<int32_t>(2 * (size_t)B);
    int64_t* idx = ar.take<int64_t>(2 * (size_t)B * L.cap_q);
    double* dist = ar.take<double>(2 * (size_t)B * L.cap_q);
    const size_t nn_bytes = feature_nn_workspace(2 * (int64_t)B, L.cap_q, L.cap_s);
    void* nn_ws = ar.take<char>(nn_bytes);
    GEOB_REQUIRE(ar.ok(), "rpmnet_metrics_batched: workspace accounting error");
    cudaStream_t st = (cudaStream_t)stream;
    int launches = 0;
    rp_pair_kernel<<<1, 32, 0, st>>>(B, gt_transforms, est_transforms, xf, out);
    const int rows = L.cap_q > L.cap_s ? L.cap_q : L.cap_s;
    rp_points_kernel<<<dim3((rows + RP_THREADS - 1) / RP_THREADS, B), RP_THREADS, 0, st>>>(L, raw, ref, src, xf, Q, S, nq, ns);
    GEOB_CHECK_LAUNCH();
    launches += 2;
    if (feature_nn_launch(Q, S, 2 * B, L.cap_q, L.cap_s, 3, nq, ns, idx, dist, nullptr, nullptr, nn_ws, nn_bytes, st, &launches)) return -1;
    rp_reduce_kernel<<<B, RP_THREADS, 0, st>>>(B, L.cap_q, nq, dist, out);
    GEOB_CHECK_LAUNCH();
    count_launches(launches + 1);
    return 0;
}

}  // extern "C"
