// Coarse (superpoint) matching, patch gathering + fine matching scores, log-domain Sinkhorn with dustbins.
//
// Reference:
//   geotransformer/modules/geotransformer/superpoint_matching.py:13-50
//   experiments/*/model.py:105-108,169-188 (patch gathers and the 'bnd,bmd->bnm' einsum / sqrt(C))
//   geotransformer/modules/sinkhorn/learnable_sinkhorn.py:13-66 (100 Python-loop iterations, ~600 launches)
// Here the 100 Sinkhorn iterations of one patch pair run inside one CTA with the (K+1)x(K+1) score matrix in
// shared memory; nothing but the input scores and the final log-assignment touches HBM.
#include "common.cuh"
#include "geob200.h"

namespace geob200 {

int segs_from_counts(Segs* s, int64_t n, const int64_t* counts) {
    if (n < 1 || n > GEOB_MAX_CLOUDS) { set_error("batch: 1..%d segments supported (got %lld)", GEOB_MAX_CLOUDS, (long long)n); return -1; }
    *s = Segs{};
    s->n = (int)n;
    int64_t o = 0;
    for (int i = 0; i < n; ++i) {
        if (counts[i] < 0) { set_error("batch: negative segment size"); return -1; }
        s->start[i] = (int)o;
        s->count[i] = (int)counts[i];
        s->max = s->max > (int)counts[i] ? s->max : (int)counts[i];
        o += counts[i];
    }
    if (o >= (1ll << 31)) { set_error("batch: too many rows (%lld)", (long long)o); return -1; }
    return 0;
}

Segs segs_one(int64_t count) {
    Segs s{};
    s.n = 1;
    s.max = (int)count;
    s.count[0] = (int)count;
    return s;
}

Segs segs_range(const Segs& s, int first, int n) {
    Segs r{};
    r.n = n;
    for (int i = 0; i < n; ++i) {
        r.start[i] = s.start[first + i];
        r.count[i] = s.count[first + i];
        r.max = r.max > r.count[i] ? r.max : r.count[i];
    }
    return r;
}

int segs_products(Segs* s, const Segs& ref, const Segs& src) {
    int64_t c[GEOB_MAX_CLOUDS];
    for (int i = 0; i < ref.n; ++i) c[i] = (int64_t)ref.count[i] * src.count[i];
    return segs_from_counts(s, ref.n, c);
}

// ---- superpoint matching ---------------------------------------------------------------------------------

// valid (non-empty) node lists, in index order (torch.nonzero): one CTA per cloud, chunked ordered compaction.  Clouds s < B are
// the ref clouds, read from ref_masks at cl.start[s]; the others from src_masks, whose block starts at cloud B.  NULL masks = all
// valid.  idx / count are stacked over all 2B clouds.
__global__ void __launch_bounds__(1024) compact_masks_kernel(const unsigned char* __restrict__ ref_masks,
                                                             const unsigned char* __restrict__ src_masks, const __grid_constant__ Segs cl,
                                                             int B, int* __restrict__ idx, int* __restrict__ count) {
    const int s = blockIdx.y;
    const unsigned char* __restrict__ masks = s < B ? ref_masks : src_masks;
    if (masks != nullptr) masks += s < B ? cl.start[s] : cl.start[s] - cl.start[B];
    idx += cl.start[s];
    count += s;
    const int n = cl.count[s];
    __shared__ int warp_tot[32];
    __shared__ int carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const int f = (i < n && (masks == nullptr || masks[i])) ? 1 : 0;
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        const int pre = __popc(bal & ((1u << lane) - 1u));
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        int off = carry;
        for (int w = 0; w < warp; ++w) off += warp_tot[w];
        if (f) idx[off + pre] = i;
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int w = 0; w < 32; ++w) t += warp_tot[w];
            carry += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = carry;
}

// S[i][j] = exp(-clamp(2 - 2 <fr_i, fs_j>, 0)) over the valid nodes; row sums.  One CTA per (compacted) row.
// Pair p = blockIdx.y: ref rows at R.start[p] of fr / ridx / rowsum, src rows at Q.start[p] of fs / sidx, S at NN.start[p].
__global__ void __launch_bounds__(256) spm_scores_kernel(const float* __restrict__ fr, const float* __restrict__ fs, int C,
                                                         const int* __restrict__ ridx, const int* __restrict__ rcount,
                                                         const int* __restrict__ sidx, const int* __restrict__ scount,
                                                         const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                         const __grid_constant__ Segs NN, float* __restrict__ S, float* __restrict__ rowsum) {
    extern __shared__ float sm[];
    const int p = blockIdx.y;
    const int ld = Q.count[p];
    fr += (long long)R.start[p] * C; ridx += R.start[p]; rcount += p; rowsum += R.start[p];
    fs += (long long)Q.start[p] * C; sidx += Q.start[p]; scount += p;
    S += NN.start[p];
    float* a = sm;            // [C]
    float* srow = sm + C;     // [ld]
    const int i = blockIdx.x;
    if (i >= *rcount) return;
    const int ns = *scount;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = threadIdx.x; c < C; c += blockDim.x) a[c] = fr[(long long)ridx[i] * C + c];
    __syncthreads();
    for (int j = warp; j < ns; j += 8) {
        const float* b = fs + (long long)sidx[j] * C;
        float d = 0.f;
        for (int c = lane; c < C; c += 32) d = fmaf(a[c], b[c], d);
        d = warp_sum(d);
        if (lane == 0) {
            const float v = expf(-fmaxf(2.0f - 2.0f * d, 0.0f));
            srow[j] = v;
            S[(long long)i * ld + j] = v;
        }
    }
    __syncthreads();
    if (warp == 0) {
        float s = 0.f;
        for (int j = lane; j < ns; j += 32) s += srow[j];
        s = warp_sum(s);
        if (lane == 0) rowsum[i] = s;
    }
}

__global__ void __launch_bounds__(256) spm_colsum_kernel(const float* __restrict__ S, const int* __restrict__ rcount,
                                                         const int* __restrict__ scount, const __grid_constant__ Segs Q,
                                                         const __grid_constant__ Segs NN, float* __restrict__ colsum) {
    const int p = blockIdx.y;
    const int ld = Q.count[p];
    S += NN.start[p]; rcount += p; scount += p; colsum += Q.start[p];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *scount) return;
    const int nr = *rcount;
    float s = 0.f;
    for (int i = 0; i < nr; ++i) s += S[(long long)i * ld + j];
    colsum[j] = s;
}

// dual normalisation into a dense flat (nr*ns) array
__global__ void __launch_bounds__(256) spm_dual_kernel(const float* __restrict__ S, const int* __restrict__ rcount,
                                                       const int* __restrict__ scount, const float* __restrict__ rowsum,
                                                       const float* __restrict__ colsum, const __grid_constant__ Segs R,
                                                       const __grid_constant__ Segs Q, const __grid_constant__ Segs NN, int dual,
                                                       float* __restrict__ flat) {
    const int p = blockIdx.y;
    const int ld = Q.count[p];
    S += NN.start[p]; flat += NN.start[p]; rcount += p; scount += p; rowsum += R.start[p]; colsum += Q.start[p];
    const int nr = *rcount, ns = *scount;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)nr * ns) return;
    const int i = (int)(t / ns), j = (int)(t % ns);
    const float v = S[(long long)i * ld + j];
    flat[t] = dual ? (v / rowsum[i]) * (v / colsum[j]) : v;
}

// top-k (largest) of a flat positive array: MSB-first 8-bit radix select of the k-th value, then an ordered
// sweep that keeps everything above the threshold and the lowest-index ties, then a bitonic sort of the k winners.
// One CTA per pair p = blockIdx.y; its k_req output rows start at p * k_req.
template <int KMAX>
__global__ void __launch_bounds__(1024) topk_flat_kernel(const float* __restrict__ flat, const int* __restrict__ rcount,
                                                         const int* __restrict__ scount, int k_req, const int* __restrict__ ridx,
                                                         const int* __restrict__ sidx, const __grid_constant__ Segs R,
                                                         const __grid_constant__ Segs Q, const __grid_constant__ Segs NN,
                                                         long long* __restrict__ ref_out, long long* __restrict__ src_out,
                                                         float* __restrict__ score_out, int* __restrict__ k_out) {
    {
        const int p = blockIdx.y;
        flat += NN.start[p]; rcount += p; scount += p; ridx += R.start[p]; sidx += Q.start[p];
        ref_out += (long long)p * k_req; src_out += (long long)p * k_req; score_out += (long long)p * k_req; k_out += p;
    }
    __shared__ unsigned hist[256];
    __shared__ unsigned long long keys[KMAX];
    __shared__ unsigned prefix_s, kth_s;
    __shared__ int warp_tot[32], carry_gt, carry_eq;
    const int nr = *rcount, ns = *scount;
    const long long total = (long long)nr * ns;
    const int k = (int)min((long long)min(k_req, KMAX), total);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // rows past the number of existing candidates are padding: index -1 (gather_patches turns it into an empty patch)
    for (int i = k + threadIdx.x; i < k_req; i += blockDim.x) { ref_out[i] = -1; src_out[i] = -1; score_out[i] = 0.f; }
    if (k == 0) { if (threadIdx.x == 0) *k_out = 0; return; }
    unsigned prefix = 0, mask = 0;
    int remaining = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (long long t = threadIdx.x; t < total; t += blockDim.x) {
            const unsigned b = __float_as_uint(flat[t]);
            if ((b & mask) == prefix) atomicAdd(&hist[(b >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int rem = remaining;
            int d = 255;
            for (; d > 0; --d) {
                if ((int)hist[d] >= rem) break;
                rem -= (int)hist[d];
            }
            prefix_s = prefix | ((unsigned)d << shift);
            kth_s = (unsigned)rem;
        }
        __syncthreads();
        prefix = prefix_s;
        remaining = (int)kth_s;
        mask |= (255u << shift);
        __syncthreads();
    }
    const unsigned thr = prefix;          // bit pattern of the k-th largest value
    const int need_eq = remaining;        // how many ties at the threshold are kept (lowest flat indices)
    const int n_gt = k - need_eq;
    if (threadIdx.x == 0) { carry_gt = 0; carry_eq = 0; }
    __syncthreads();
    for (long long base = 0; base < total; base += 1024) {
        const long long t = base + threadIdx.x;
        unsigned b = 0;
        if (t < total) b = __float_as_uint(flat[t]);
        const int fg = (t < total && b > thr) ? 1 : 0;
        const int fe = (t < total && b == thr) ? 1 : 0;
        const unsigned bg = __ballot_sync(0xffffffffu, fg), be = __ballot_sync(0xffffffffu, fe);
        const int pg = __popc(bg & ((1u << lane) - 1u)), pe = __popc(be & ((1u << lane) - 1u));
        if (lane == 0) warp_tot[warp] = (__popc(bg) << 16) | __popc(be);
        __syncthreads();
        int og = carry_gt, oe = carry_eq;
        for (int w = 0; w < warp; ++w) { og += warp_tot[w] >> 16; oe += warp_tot[w] & 0xFFFF; }
        const unsigned long long key = ((unsigned long long)b << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)t);
        if (fg) keys[og + pg] = key;
        if (fe && oe + pe < need_eq) keys[n_gt + oe + pe] = key;
        __syncthreads();
        if (threadIdx.x == 0) {
            int tg = 0, te = 0;
            for (int w = 0; w < 32; ++w) { tg += warp_tot[w] >> 16; te += warp_tot[w] & 0xFFFF; }
            carry_gt += tg; carry_eq += te;
        }
        __syncthreads();
    }
    int n2 = 1;
    while (n2 < k) n2 <<= 1;
    for (int i = k + threadIdx.x; i < n2; i += blockDim.x) keys[i] = 0ull;
    __syncthreads();
    for (int kk = 2; kk <= n2; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < n2; t += blockDim.x) {
                const int p = t ^ j;
                if (p > t) {
                    const unsigned long long a = keys[t], b = keys[p];
                    const bool desc = ((t & kk) == 0);
                    if ((a < b) == desc) { keys[t] = b; keys[p] = a; }
                }
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const unsigned long long key = keys[i];
        const unsigned t = 0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull);
        ref_out[i] = ridx[t / ns];
        src_out[i] = sidx[t % ns];
        score_out[i] = __uint_as_float((unsigned)(key >> 32));
    }
    if (threadIdx.x == 0) *k_out = k;
}

// ---- patch gathers ---------------------------------------------------------------------------------------
// out_idx[p][i] = knn[corr[p]][i]; out_mask likewise; out_pts = padded_points[idx].  Cloud s = blockIdx.y: its node rows
// (knn table) at Nd.start[s], its points at Pt.start[s]; P patches per cloud at s * P, or with corr == nullptr every node of the
// cloud is a patch (corr = arange), at Nd.start[s].
__global__ void __launch_bounds__(256) gather_patches_kernel(const long long* __restrict__ corr, int P_all, const long long* __restrict__ knn,
                                                             const unsigned char* __restrict__ knn_masks, int K,
                                                             const float* __restrict__ pts, const __grid_constant__ Segs Nd,
                                                             const __grid_constant__ Segs Pt, long long* __restrict__ out_idx,
                                                             unsigned char* __restrict__ out_mask, float* __restrict__ out_pts) {
    const int s = blockIdx.y;
    const int P = corr != nullptr ? P_all : Nd.count[s];
    const long long first = corr != nullptr ? (long long)s * P_all : Nd.start[s];
    if (corr != nullptr) corr += first;
    knn += (long long)Nd.start[s] * K; knn_masks += (long long)Nd.start[s] * K;
    pts += 3ll * Pt.start[s];
    const int n_pts = Pt.count[s];
    out_idx += first * K; out_mask += first * K; out_pts += 3 * first * K;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P * K) return;
    const int p = t / K, i = t % K;
    const long long node = corr != nullptr ? corr[p] : p;
    const long long idx = node >= 0 ? knn[node * K + i] : (long long)n_pts;
    out_idx[t] = idx;
    out_mask[t] = node >= 0 ? knn_masks[node * K + i] : 0;
    const bool ok = idx < n_pts;
    out_pts[3 * t + 0] = ok ? pts[3 * idx + 0] : 0.f;
    out_pts[3 * t + 1] = ok ? pts[3 * idx + 1] : 0.f;
    out_pts[3 * t + 2] = ok ? pts[3 * idx + 2] : 0.f;
}

// scores[p][i][j] = <fr[ridx[p][i]], fs[sidx[p][j]]> / sqrt(C); rows of the sentinel index are zero.
// One CTA per patch; T = K/16 outputs per thread per dimension.
// Pair b = blockIdx.y: ref fine rows at R.start[b] of fr, src at Q.start[b] of fs; patches b * gridDim.x + blockIdx.x.
template <int T>
__global__ void __launch_bounds__(256) patch_scores_kernel(const float* __restrict__ fr, const float* __restrict__ fs,
                                                           const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                           int C, const long long* __restrict__ ridx, const long long* __restrict__ sidx,
                                                           float inv_div, float* __restrict__ out) {
    constexpr int K = 16 * T, CH = 32;
    __shared__ float A[K][CH + 1], B[K][CH + 1];
    const int b = blockIdx.y;
    fr += (long long)R.start[b] * C; fs += (long long)Q.start[b] * C;
    const int nr = R.count[b], ns = Q.count[b];
    const int p = b * gridDim.x + blockIdx.x;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[T][T];
#pragma unroll
    for (int a = 0; a < T; ++a)
#pragma unroll
        for (int b = 0; b < T; ++b) acc[a][b] = 0.f;
    for (int c0 = 0; c0 < C; c0 += CH) {
        for (int e = threadIdx.x; e < K * CH; e += 256) {
            const int r = e / CH, c = e % CH;
            const long long ia = ridx[(long long)p * K + r], ib = sidx[(long long)p * K + r];
            A[r][c] = (ia < nr && c0 + c < C) ? fr[ia * C + c0 + c] : 0.f;
            B[r][c] = (ib < ns && c0 + c < C) ? fs[ib * C + c0 + c] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int c = 0; c < CH; ++c) {
            float av[T], bv[T];
#pragma unroll
            for (int a = 0; a < T; ++a) av[a] = A[ty + 16 * a][c];
#pragma unroll
            for (int b = 0; b < T; ++b) bv[b] = B[tx + 16 * b][c];
#pragma unroll
            for (int a = 0; a < T; ++a)
#pragma unroll
                for (int b = 0; b < T; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < T; ++a)
#pragma unroll
        for (int b = 0; b < T; ++b)
            out[((long long)p * K + ty + 16 * a) * K + tx + 16 * b] = acc[a][b] / inv_div;
}

// ---- Sinkhorn --------------------------------------------------------------------------------------------
// One CTA per patch pair.  Z (K+1)x(K+1) padded scores in shared memory, row/col potentials u, v.
// learnable_sinkhorn.py:13-18:  u = log_mu - LSE_j(Z + v) ; v = log_nu - LSE_i(Z + u)   x num_iterations
__global__ void __launch_bounds__(1024) sinkhorn_kernel(const float* __restrict__ scores, const unsigned char* __restrict__ row_masks,
                                                       const unsigned char* __restrict__ col_masks, const float* __restrict__ alpha_p,
                                                       int K, int iters, float inf, float* __restrict__ out) {
    extern __shared__ float sm[];
    const int K1 = K + 1;
    const int ld = K1 | 1;                   // odd row stride: conflict-free column walks
    float* Z = sm;                           // [K1][ld]
    float* u = Z + K1 * ld;
    float* v = u + K1;
    float* lmu = v + K1;
    float* lnu = lmu + K1;
    __shared__ float norm_s;
    __shared__ int cnt_s[2];
    const int p = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float alpha = *alpha_p;
    if (threadIdx.x < 2) cnt_s[threadIdx.x] = 0;
    __syncthreads();
    {
        int cr = 0, cc = 0;
        for (int i = threadIdx.x; i < K; i += blockDim.x) { cr += row_masks[(long long)p * K + i] ? 1 : 0; cc += col_masks[(long long)p * K + i] ? 1 : 0; }
        atomicAdd(&cnt_s[0], cr);
        atomicAdd(&cnt_s[1], cc);
    }
    __syncthreads();
    const float nvr = (float)cnt_s[0], nvc = (float)cnt_s[1];
    if (threadIdx.x == 0) norm_s = -logf(nvr + nvc);
    __syncthreads();
    const float norm = norm_s;
    for (int e = threadIdx.x; e < K1 * K1; e += blockDim.x) {
        const int i = e / K1, j = e % K1;
        float z = (i < K && j < K) ? scores[((long long)p * K + i) * K + j] : alpha;
        const bool rm = (i < K) && !row_masks[(long long)p * K + i];
        const bool cm = (j < K) && !col_masks[(long long)p * K + j];
        if (rm || cm) z = -inf;
        Z[i * ld + j] = z;
    }
    for (int i = threadIdx.x; i < K1; i += blockDim.x) {
        float mu = (i < K) ? norm : logf(nvc) + norm;
        float nu = (i < K) ? norm : logf(nvr) + norm;
        if (i < K && !row_masks[(long long)p * K + i]) mu = -inf;
        if (i < K && !col_masks[(long long)p * K + i]) nu = -inf;
        lmu[i] = mu; lnu[i] = nu; u[i] = 0.f; v[i] = 0.f;
    }
    __syncthreads();
    // 8 lanes per row/column (4 rows per warp at once): 3-step shuffle reductions and ~K/8 independent exp per lane keep the
    // dependent chain of one half-iteration short (the kernel is latency-, not throughput-bound)
    const int nslot = (blockDim.x >> 5) * 4;
    const int grp = lane >> 3, sub = lane & 7;
    for (int it = 0; it < iters; ++it) {
        for (int base = warp * 4; base < K1; base += nslot) {     // warp-uniform trip count: every lane joins the shuffles
            const bool act = base + grp < K1;
            const int i = act ? base + grp : K1 - 1;
            const float* zr = Z + i * ld;
            float mx = -INFINITY;
            for (int j = sub; j < K1; j += 8) mx = fmaxf(mx, zr[j] + v[j]);
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float s = 0.f;
            for (int j = sub; j < K1; j += 8) s += expf(zr[j] + v[j] - mx);
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (act && sub == 0) u[i] = lmu[i] - (logf(s) + mx);
        }
        __syncthreads();
        for (int base = warp * 4; base < K1; base += nslot) {
            const bool act = base + grp < K1;
            const int j = act ? base + grp : K1 - 1;
            float mx = -INFINITY;
            for (int i = sub; i < K1; i += 8) mx = fmaxf(mx, Z[i * ld + j] + u[i]);
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float s = 0.f;
            for (int i = sub; i < K1; i += 8) s += expf(Z[i * ld + j] + u[i] - mx);
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (act && sub == 0) v[j] = lnu[j] - (logf(s) + mx);
        }
        __syncthreads();
    }
    for (int e = threadIdx.x; e < K1 * K1; e += blockDim.x) {
        const int i = e / K1, j = e % K1;
        out[(long long)p * K1 * K1 + e] = Z[i * ld + j] + u[i] + v[j] - norm;
    }
}

// Register-resident variant (K+1 <= MAXT / LPR rows): every thread keeps its NE entries of its row AND its NE entries of its
// column in registers for all iterations, in the log2 domain (Z * log2 e), so that a half-iteration is one shared-memory load
// (the other potential), one ex2 and ~4 ALU instructions per entry.  The generic kernel above re-reads Z from shared memory
// twice per entry and pays expf's range reduction; it is issue-bound at 64 resident warps per SM.
template <int LPR, int NE, int MAXT>
__global__ void __launch_bounds__(MAXT) sinkhorn_reg_kernel(const float* __restrict__ scores, const unsigned char* __restrict__ row_masks,
                                                           const unsigned char* __restrict__ col_masks, const float* __restrict__ alpha_p,
                                                           int K, int iters, float inf, float* __restrict__ out) {
    extern __shared__ float sm[];
    const int K1 = K + 1;
    const int ld = K1 | 1;
    float* Z = sm;                           // [K1][ld], natural-log domain (also the source of the final output)
    float* u = Z + K1 * ld;                  // log2 domain
    float* v = u + K1;
    __shared__ float norm_s;
    __shared__ int cnt_s[2];
    const int p = blockIdx.x;
    const float alpha = *alpha_p;
    constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
    if (threadIdx.x < 2) cnt_s[threadIdx.x] = 0;
    __syncthreads();
    {
        int cr = 0, cc = 0;
        for (int i = threadIdx.x; i < K; i += blockDim.x) { cr += row_masks[(long long)p * K + i] ? 1 : 0; cc += col_masks[(long long)p * K + i] ? 1 : 0; }
        if (cr) atomicAdd(&cnt_s[0], cr);
        if (cc) atomicAdd(&cnt_s[1], cc);
    }
    __syncthreads();
    const float nvr = (float)cnt_s[0], nvc = (float)cnt_s[1];
    if (threadIdx.x == 0) norm_s = -logf(nvr + nvc);
    __syncthreads();
    const float norm = norm_s;
    for (int e = threadIdx.x; e < K1 * K1; e += blockDim.x) {
        const int i = e / K1, j = e % K1;
        float z = (i < K && j < K) ? scores[((long long)p * K + i) * K + j] : alpha;
        const bool rm = (i < K) && !row_masks[(long long)p * K + i];
        const bool cm = (j < K) && !col_masks[(long long)p * K + j];
        if (rm || cm) z = -inf;
        Z[i * ld + j] = z;
    }
    for (int i = threadIdx.x; i < K1; i += blockDim.x) { u[i] = 0.f; v[i] = 0.f; }
    __syncthreads();
    const int slot = threadIdx.x / LPR, sub = threadIdx.x % LPR;
    const bool act = slot < K1;
    const int ij = act ? slot : K1 - 1;
    float zr[NE], zc[NE];
#pragma unroll
    for (int k = 0; k < NE; ++k) {
        const int o = sub + LPR * k;
        zr[k] = (o < K1) ? Z[ij * ld + o] * LOG2E : -INFINITY;      // row ij, column o
        zc[k] = (o < K1) ? Z[o * ld + ij] * LOG2E : -INFINITY;      // column ij, row o
    }
    float lmu2, lnu2;                                               // log2-domain marginals of row / column ij
    {
        float mu = (ij < K) ? norm : logf(nvc) + norm;
        float nu = (ij < K) ? norm : logf(nvr) + norm;
        if (ij < K && !row_masks[(long long)p * K + ij]) mu = -inf;
        if (ij < K && !col_masks[(long long)p * K + ij]) nu = -inf;
        lmu2 = mu * LOG2E;
        lnu2 = nu * LOG2E;
    }
    for (int it = 0; it < iters; ++it) {
        {
            float t[NE], mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < NE; ++k) {
                const int o = sub + LPR * k;
                t[k] = zr[k] + v[o < K1 ? o : 0];
                mx = fmaxf(mx, t[k]);
            }
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < NE; ++k) s += exp2f(t[k] - mx);
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (act && sub == 0) u[ij] = lmu2 - (log2f(s) + mx);
        }
        __syncthreads();
        {
            float t[NE], mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < NE; ++k) {
                const int o = sub + LPR * k;
                t[k] = zc[k] + u[o < K1 ? o : 0];
                mx = fmaxf(mx, t[k]);
            }
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < NE; ++k) s += exp2f(t[k] - mx);
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (act && sub == 0) v[ij] = lnu2 - (log2f(s) + mx);
        }
        __syncthreads();
    }
    for (int e = threadIdx.x; e < K1 * K1; e += blockDim.x) {
        const int i = e / K1, j = e % K1;
        out[(long long)p * K1 * K1 + e] = Z[i * ld + j] + (u[i] + v[j]) * LN2 - norm;
    }
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_superpoint_matching_batched_workspace_bytes(int64_t n_rows, int64_t n_products, int64_t n_pairs) {
    const size_t r = (size_t)n_rows, nn = (size_t)n_products;
    return align_up(4 * r, 256) * 3 + align_up(4 * nn, 256) * 2 + align_up(8 * (size_t)n_pairs, 256) + 4096;
}

int geob200_superpoint_matching_batched(const float* ref_feats, const float* src_feats, int64_t channels, const uint8_t* ref_masks,
                                        const uint8_t* src_masks, int64_t n_pairs, const int64_t* cloud_nodes, int64_t num_correspondences,
                                        int dual, int64_t* corr_indices, float* corr_scores, int32_t* num_out, void* workspace,
                                        size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "superpoint_matching_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(num_correspondences > 0 && num_correspondences <= 1024, "superpoint_matching: num_correspondences must be in 1..1024");
    const int B = (int)n_pairs;
    // cl: all 2B clouds stacked (the workspace rows); R / Q: the ref / src clouds in the row spaces of ref_feats / src_feats
    Segs cl, Q, NN;
    if (segs_from_counts(&cl, 2 * n_pairs, cloud_nodes) || segs_from_counts(&Q, n_pairs, cloud_nodes + n_pairs)) return -1;
    const Segs R = segs_range(cl, 0, B);
    const int64_t ref_rows = cl.start[B], rows = (int64_t)cl.start[2 * B - 1] + cl.count[2 * B - 1];
    GEOB_REQUIRE(ref_rows > 0 && rows > ref_rows, "superpoint_matching: empty input");
    if (segs_products(&NN, R, Q)) return -1;
    const int64_t nn = (int64_t)NN.start[B - 1] + NN.count[B - 1];
    GEOB_REQUIRE(workspace_bytes >= geob200_superpoint_matching_batched_workspace_bytes(rows, nn, n_pairs),
                 "superpoint_matching_batched: workspace too small");
    const size_t smem = sizeof(float) * (channels + Q.max);
    GEOB_REQUIRE(smem <= 48 * 1024, "superpoint_matching: row does not fit shared memory");
    Arena ar(workspace, workspace_bytes);
    int* idx = ar.take<int>(rows);               // ref clouds' valid nodes, then the src clouds' (at ref_rows)
    float* rowsum = ar.take<float>(rows);
    float* colsum = ar.take<float>(rows);
    float* S = ar.take<float>(nn);
    float* flat = ar.take<float>(nn);
    int* counts = ar.take<int>(2 * B);           // counts[p] / counts[B + p] = valid ref / src nodes of pair p
    const int* ridx = idx;
    const int* sidx = idx + ref_rows;
    const dim3 g_rows((unsigned)(R.max > 0 ? R.max : 1), B), g_cols((unsigned)((Q.max + 255) / 256 > 0 ? (Q.max + 255) / 256 : 1), B),
        g_nn((unsigned)((NN.max + 255) / 256 > 0 ? (NN.max + 255) / 256 : 1), B);
    const int64_t k = num_correspondences;
    compact_masks_kernel<<<dim3(1, 2 * B), 1024, 0, st>>>(ref_masks, src_masks, cl, B, idx, counts);
    spm_scores_kernel<<<g_rows, 256, smem, st>>>(ref_feats, src_feats, (int)channels, ridx, counts, sidx, counts + B, R, Q, NN, S, rowsum);
    spm_colsum_kernel<<<g_cols, 256, 0, st>>>(S, counts, counts + B, Q, NN, colsum);
    spm_dual_kernel<<<g_nn, 256, 0, st>>>(S, counts, counts + B, rowsum, colsum, R, Q, NN, dual, flat);
    topk_flat_kernel<1024><<<dim3(1, B), 1024, 0, st>>>(flat, counts, counts + B, (int)k, ridx, sidx, R, Q, NN, (long long*)corr_indices,
                                                        (long long*)corr_indices + B * k, corr_scores, num_out);
    GEOB_CHECK_LAUNCH();
    count_launches(5);
    return 0;
}

int geob200_gather_patches_batched(const int64_t* corr_indices, int64_t n_corr, int64_t n_clouds, const int64_t* cloud_nodes,
                                   const int64_t* cloud_points, const int64_t* node_knn_indices, const uint8_t* node_knn_masks, int64_t k,
                                   const float* points, int64_t* out_indices, uint8_t* out_masks, float* out_points, void* stream) {
    Segs nd, pt;
    if (segs_from_counts(&nd, n_clouds, cloud_nodes) || segs_from_counts(&pt, n_clouds, cloud_points)) return -1;
    const int64_t per = corr_indices != nullptr ? n_corr : nd.max;
    if (per == 0) return 0;
    gather_patches_kernel<<<dim3((unsigned)((per * k + 255) / 256), (unsigned)n_clouds), 256, 0, (cudaStream_t)stream>>>(
        (const long long*)corr_indices, (int)n_corr, (const long long*)node_knn_indices, node_knn_masks, (int)k, points, nd, pt,
        (long long*)out_indices, out_masks, out_points);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_patch_scores_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs, const int64_t* cloud_points,
                                 const int64_t* ref_knn_indices, const int64_t* src_knn_indices, int64_t n_patches, int64_t k,
                                 float* scores, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "patch_scores_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    Segs R, Q;
    if (segs_from_counts(&R, n_pairs, cloud_points) || segs_from_counts(&Q, n_pairs, cloud_points + n_pairs)) return -1;
    if (n_patches == 0) return 0;
    const float div = sqrtf((float)channels);      // feats_f.shape[1] ** 0.5
    const dim3 grid((unsigned)n_patches, R.n);
#define LAUNCH_PS(TV) patch_scores_kernel<TV><<<grid, 256, 0, st>>>(ref_feats, src_feats, R, Q, (int)channels,                      \
                                                                    (const long long*)ref_knn_indices, (const long long*)src_knn_indices, div, scores)
    if (k == 64) LAUNCH_PS(4);
    else if (k == 128) LAUNCH_PS(8);
    else if (k == 32) LAUNCH_PS(2);
    else
        GEOB_REQUIRE(false, "patch_scores: num_points_in_patch=%lld unsupported (32, 64, 128)", (long long)k);
#undef LAUNCH_PS
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_sinkhorn(const float* scores, const uint8_t* row_masks, const uint8_t* col_masks, const float* alpha,
                     int64_t n_patches, int64_t k, int64_t num_iterations, float inf, float* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (n_patches == 0) return 0;
    const int K1 = (int)k + 1, ld = K1 | 1;
    const size_t smem = sizeof(float) * ((size_t)K1 * ld + 4 * K1);
    GEOB_REQUIRE(smem <= 200 * 1024, "sinkhorn: patch too large (k=%lld)", (long long)k);
    if (smem > 48 * 1024 && ensure_max_smem((const void*)sinkhorn_kernel)) return -1;
#define LAUNCH_SK_REG(LPRV, NEV, MT)                                                                                                  \
    {                                                                                                                            \
        if (smem > 48 * 1024 && ensure_max_smem((const void*)sinkhorn_reg_kernel<LPRV, NEV, MT>)) return -1;                         \
        const int threads = ((K1 * LPRV + 31) / 32) * 32;                                                                        \
        sinkhorn_reg_kernel<LPRV, NEV, MT><<<(unsigned)n_patches, threads, smem, st>>>(scores, row_masks, col_masks, alpha, (int)k,  \
                                                                                  (int)num_iterations, inf, out);               \
    }
    if (K1 <= 40) LAUNCH_SK_REG(8, 5, 320)
    else if (K1 <= 72) LAUNCH_SK_REG(8, 9, 576)
    else if (K1 <= 132) LAUNCH_SK_REG(4, 33, 544)
    else
        sinkhorn_kernel<<<(unsigned)n_patches, 1024, smem, st>>>(scores, row_masks, col_masks, alpha, (int)k, (int)num_iterations, inf, out);
#undef LAUNCH_SK_REG
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
