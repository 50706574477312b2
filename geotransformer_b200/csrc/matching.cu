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

// ---- Sinkhorn backward -----------------------------------------------------------------------------------
// Reverse sweep of learnable_sinkhorn.py:13-18 for one patch per CTA, same ownership as sinkhorn_reg_kernel: thread (slot, sub) owns
// the entries (slot, sub + LPR k) of row `slot` and (sub + LPR k, slot) of column `slot`; Z stays in shared memory and dZ of a thread's
// row entries in registers.  The row half-step's terms (computed by the column owners) pass through shared memory (D) and are added
// by the row owners before the next column half-step, so dZ accumulates G, then the terms of iteration T, T-1, ... in autograd's order:
// the running sum stays small (two separate accumulators would each grow to ~iters terms and cancel only at the end).  The CTA first re-runs the forward iterations and streams the log-sum-exp of every half-step (Lu_t, Lv_t,
// t = 1..iters) to its slice of `hist`; the reverse sweep reads them back from the last iteration to the first:
//   column half-step (row owners):    P^v_ij = exp(x^v_ij - Lv_j),  dZ_ij -= gv_j P^v_ij,  gu_i = [t = T] rowsum(G)_i - sum_j gv_j P^v_ij
//   row half-step (column owners):    P^u_ij = exp(x^u_ij - Lu_i),  dZ_ij -= gu_i P^u_ij,  gv_j = -sum_i gu_i P^u_ij
// with the logits x^v_ij = Z_ij + u_i, x^u_ij = Z_ij + v_j.  A masked line (row or column whose mask is false) is -inf on all its
// entries; the logits of such a line drop the constant (x^u_ij = v_j on a masked row, x^v_ij = u_i on a masked column) and its
// potential is -L instead of log_mu - L: the inf -> infinity limit of the reference's arithmetic, which fp64 autograd follows and fp32
// loses (1e12 swallows the potentials).  So an upstream gradient on masked entries stays finite.  The output gradient is zero on masked
// entries (masked_fill); dalpha_part[p] = the sum of dZ over the unmasked dustbin entries.  A padding patch (no valid row and no valid
// column) writes zeros and a zero partial.
template <int K, int LPR, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) sinkhorn_bwd_kernel(const float* __restrict__ scores, const unsigned char* __restrict__ row_masks,
                                                           const unsigned char* __restrict__ col_masks, const float* __restrict__ alpha_p,
                                                           int iters, float inf, const float* __restrict__ grad,
                                                           float* __restrict__ hist, float* __restrict__ dscores,
                                                           float* __restrict__ dalpha_part) {
    constexpr int K1 = K + 1, ld = K1 | 1, NE = (K1 + LPR - 1) / LPR;
    extern __shared__ float sm[];
    float* Z = sm;                           // [K1][ld]; after the sweep: the accumulated dZ
    float* D = Z + K1 * ld;                  // [K1][ld]: the last row half-step's dZ terms
    float* pu = D + K1 * ld;                 // u_t
    float* pv = pu + K1;                     // v_t (forward), v_{t-1} (sweep)
    float* Lu = pv + K1;
    float* Lv = Lu + K1;
    float* gu = Lv + K1;
    float* gv = gu + K1;
    unsigned char* rmk = reinterpret_cast<unsigned char*>(gv + K1);     // row i is masked (all -inf)
    unsigned char* cmk = rmk + K1;
    __shared__ int cnt_s[2];
    const int p = blockIdx.x;
    row_masks += (long long)p * K; col_masks += (long long)p * K;
    grad += (long long)p * K1 * K1;
    hist += (long long)p * 2 * iters * K1;
    dscores += (long long)p * K * K;
    if (threadIdx.x < 2) cnt_s[threadIdx.x] = 0;
    __syncthreads();
    {
        int cr = 0, cc = 0;
        for (int i = threadIdx.x; i < K; i += blockDim.x) { cr += row_masks[i] ? 1 : 0; cc += col_masks[i] ? 1 : 0; }
        if (cr) atomicAdd(&cnt_s[0], cr);
        if (cc) atomicAdd(&cnt_s[1], cc);
    }
    __syncthreads();
    const int nr = cnt_s[0], nc = cnt_s[1];
    if (nr == 0 && nc == 0) {
        for (int e = threadIdx.x; e < K * K; e += blockDim.x) dscores[e] = 0.f;
        if (threadIdx.x == 0) dalpha_part[p] = 0.f;
        return;
    }
    const float nvr = (float)nr, nvc = (float)nc;
    const float norm = -logf(nvr + nvc);
    const float alpha = *alpha_p;
    for (int e = threadIdx.x; e < K1 * K1; e += blockDim.x) {
        const int i = e / K1, j = e % K1;
        float z = (i < K && j < K) ? scores[((long long)p * K + i) * K + j] : alpha;
        if ((i < K && !row_masks[i]) || (j < K && !col_masks[j])) z = -inf;
        Z[i * ld + j] = z;
        D[i * ld + j] = 0.f;
    }
    for (int i = threadIdx.x; i < K1; i += blockDim.x) {
        rmk[i] = i < K && !row_masks[i];
        cmk[i] = i < K && !col_masks[i];
        pu[i] = 0.f; pv[i] = 0.f;
    }
    __syncthreads();
    // marginals of unmasked lines (a masked line's potential does not use them)
    auto lmu = [&](int i) { return i < K ? norm : logf(nvc) + norm; };
    auto lnu = [&](int j) { return j < K ? norm : logf(nvr) + norm; };
    const int slot = threadIdx.x / LPR, sub = threadIdx.x % LPR;
    const bool act = slot < K1;
    const int ij = act ? slot : K1 - 1;
    const bool rm_own = rmk[ij], cm_own = cmk[ij];
    // line log-sum-exp over this thread's entries + the LPR-lane shuffle reduction
    auto lse = [&](const float (&x)[NE]) {
        float mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < NE; ++k) mx = fmaxf(mx, x[k]);
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NE; ++k) s += expf(x[k] - mx);
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        return mx + logf(s);
    };
    auto lane_sum = [&](float s) {
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        return s;
    };
    // ---- forward re-run: the log-sum-exp history
    for (int it = 0; it < iters; ++it) {
        {
            float x[NE];
#pragma unroll
            for (int k = 0; k < NE; ++k) {
                const int o = sub + LPR * k;
                x[k] = o < K1 ? (rm_own ? pv[o] : Z[ij * ld + o] + pv[o]) : -INFINITY;
            }
            const float L = lse(x);
            if (act && sub == 0) {
                hist[(long long)it * 2 * K1 + ij] = L;
                pu[ij] = rm_own ? -L : lmu(ij) - L;
            }
        }
        __syncthreads();
        {
            float x[NE];
#pragma unroll
            for (int k = 0; k < NE; ++k) {
                const int o = sub + LPR * k;
                x[k] = o < K1 ? (cm_own ? pu[o] : Z[o * ld + ij] + pu[o]) : -INFINITY;
            }
            const float L = lse(x);
            if (act && sub == 0) {
                hist[(long long)it * 2 * K1 + K1 + ij] = L;
                pv[ij] = cm_own ? -L : lnu(ij) - L;
            }
        }
        __syncthreads();
    }
    // ---- reverse sweep
    float dz[NE];                            // dZ of my row entries, starting from G
    {
        float sr = 0.f, sc = 0.f;
#pragma unroll
        for (int k = 0; k < NE; ++k) {
            const int o = sub + LPR * k;
            dz[k] = o < K1 ? grad[(long long)ij * K1 + o] : 0.f;
            if (o < K1) { sr += dz[k]; sc += grad[(long long)o * K1 + ij]; }
        }
        sr = lane_sum(sr);
        sc = lane_sum(sc);
        if (act && sub == 0) { gu[ij] = sr; gv[ij] = sc; }
    }
    for (int it = iters - 1; it >= 0; --it) {
        const float* h = hist + (long long)it * 2 * K1;
        for (int i = threadIdx.x; i < K1; i += blockDim.x) {
            const float lu = h[i], lv = h[K1 + i];
            Lu[i] = lu; Lv[i] = lv;
            pu[i] = rmk[i] ? -lu : lmu(i) - lu;
            pv[i] = it == 0 ? 0.f : (cmk[i] ? -h[K1 + i - 2 * K1] : lnu(i) - h[K1 + i - 2 * K1]);
        }
        __syncthreads();
        {   // column half-step of iteration it (v_t = log_nu - LSE_i(Z + u_t)), row owners
            const float ui = pu[ij];
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < NE; ++k) {
                const int o = sub + LPR * k;
                if (o < K1) {
                    dz[k] += D[ij * ld + o];        // the row half-step of iteration it + 1 (zero before the last iteration)
                    const float x = cmk[o] ? ui : Z[ij * ld + o] + ui;
                    const float w = gv[o] * expf(x - Lv[o]);
                    dz[k] -= w;
                    s += w;
                }
            }
            s = lane_sum(s);
            if (act && sub == 0) gu[ij] = (it == iters - 1 ? gu[ij] : 0.f) - s;
        }
        __syncthreads();
        {   // row half-step (u_t = log_mu - LSE_j(Z + v_{t-1})), column owners
            const float vj = pv[ij];
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < NE; ++k) {
                const int o = sub + LPR * k;
                if (o < K1) {
                    const float x = rmk[o] ? vj : Z[o * ld + ij] + vj;
                    const float w = gu[o] * expf(x - Lu[o]);
                    D[o * ld + ij] = -w;
                    s += w;
                }
            }
            s = lane_sum(s);
            if (act && sub == 0) gv[ij] = -s;
        }
        __syncthreads();
    }
    // the first iteration's row half-step, then dZ into Z's storage
#pragma unroll
    for (int k = 0; k < NE; ++k) {
        const int o = sub + LPR * k;
        if (act && o < K1) Z[ij * ld + o] = dz[k] + D[ij * ld + o];
    }
    __syncthreads();
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
        const int i = e / K, j = e % K;
        dscores[e] = (rmk[i] || cmk[j]) ? 0.f : Z[i * ld + j];
    }
    if (threadIdx.x < 32) {
        float s = 0.f;
        for (int e = threadIdx.x; e < 2 * K + 1; e += 32) {
            const int i = e < K ? e : K, j = e < K ? K : e - K;     // (e, K) for e < K, then (K, e - K) for e - K in 0..K
            if (!rmk[i] && !cmk[j]) s += Z[i * ld + j];
        }
        s = warp_sum(s);
        if (threadIdx.x == 0) dalpha_part[p] = s;
    }
}

// out[0] = sum of the n partials in a fixed order (thread-strided sums, then a fixed tree): deterministic for a given n
__global__ void __launch_bounds__(256) sum_partials_kernel(const float* __restrict__ part, int n, float* __restrict__ out) {
    __shared__ float red[8];
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) s += part[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w];
        out[0] = t;
    }
}

// ---- patch-score backward --------------------------------------------------------------------------------
// Per (patch, slot) gradient rows: side 0 (blockIdx.z): tmp[p K + a] = sum_b (dS_p[a][b] / sqrt(C)) fs[sidx[p][b]]; side 1:
// tmp[P_all K + p K + b] = sum_a (dS_p[a][b] / sqrt(C)) fr[ridx[p][a]].  Sentinel rows read as zero.  One CTA per patch and side,
// dS_p (transposed for side 1) in shared memory; each thread owns K/32 rows x 4 channels of a 32-channel chunk.
template <int K>
__global__ void __launch_bounds__(256) patch_scores_bwd_kernel(const float* __restrict__ fr, const float* __restrict__ fs,
                                                               const __grid_constant__ Segs R, const __grid_constant__ Segs Q, int C,
                                                               const long long* __restrict__ ridx, const long long* __restrict__ sidx,
                                                               float div, const float* __restrict__ dS, float* __restrict__ tmp) {
    constexpr int CH = 32, RT = K / 32;
    extern __shared__ float sm[];
    float* D = sm;                           // [K][K + 1]
    float* F = sm + K * (K + 1);             // [K][CH + 1]
    const int side = blockIdx.z, b = blockIdx.y;
    const long long p = (long long)b * gridDim.x + blockIdx.x;
    const long long P_all = (long long)gridDim.x * gridDim.y;
    const float* other = side ? fr + (long long)R.start[b] * C : fs + (long long)Q.start[b] * C;
    const int n_other = side ? R.count[b] : Q.count[b];
    const long long* idx = (side ? ridx : sidx) + p * K;
    dS += p * K * K;
    tmp += ((long long)side * P_all + p) * K * C;
    for (int e = threadIdx.x; e < K * K; e += 256) {
        const int a = e / K, c = e % K;
        const float g = dS[e] / div;
        if (side) D[c * (K + 1) + a] = g; else D[a * (K + 1) + c] = g;
    }
    const int ty = threadIdx.x >> 3, tx = threadIdx.x & 7;
    for (int c0 = 0; c0 < C; c0 += CH) {
        for (int e = threadIdx.x; e < K * CH; e += 256) {
            const int r = e / CH, c = e % CH;
            const long long id = idx[r];
            F[r * (CH + 1) + c] = (id >= 0 && id < n_other && c0 + c < C) ? other[id * C + c0 + c] : 0.f;
        }
        __syncthreads();
        float acc[RT][4];
#pragma unroll
        for (int r = 0; r < RT; ++r)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
#pragma unroll 4
        for (int m = 0; m < K; ++m) {
            float fv[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) fv[q] = F[m * (CH + 1) + tx + 8 * q];
#pragma unroll
            for (int r = 0; r < RT; ++r) {
                const float dv = D[(ty + 32 * r) * (K + 1) + m];
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[r][q] = fmaf(dv, fv[q], acc[r][q]);
            }
        }
#pragma unroll
        for (int r = 0; r < RT; ++r)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int c = c0 + tx + 8 * q;
                if (c < C) tmp[(long long)(ty + 32 * r) * C + c] = acc[r][q];
            }
        __syncthreads();
    }
}

// Inverse index of the (side, patch, slot) entries: entry e < 2 P_all K refers to feature row row_of(e) of the stacked row space
// (ref rows, then src rows) or to nothing (sentinel).  Rows get their entries grouped by a counting sort and ordered by entry id, so
// each row's gradient is summed in (patch, slot) order: deterministic, and a pair's rows see only the pair's own patches.
struct PatchRows {
    const long long* ridx;
    const long long* sidx;
    long long per_side;                      // P_all * K
    int K, P, n_ref_rows;
    __device__ __forceinline__ int row_of(long long e, const Segs& R, const Segs& Q) const {
        const int side = e >= per_side;
        const long long r = side ? e - per_side : e;
        const int b = (int)(r / ((long long)P * K));
        const long long id = (side ? sidx : ridx)[r];
        const Segs& S = side ? Q : R;
        if (id < 0 || id >= S.count[b]) return -1;
        return (side ? n_ref_rows : 0) + S.start[b] + (int)id;
    }
};

__global__ void __launch_bounds__(256) patch_rows_count_kernel(PatchRows pr, const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                               int* __restrict__ cnt) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 2 * pr.per_side) return;
    const int row = pr.row_of(e, R, Q);
    if (row >= 0) atomicAdd(&cnt[row], 1);
}

// exclusive prefix sum of cnt[0..n) into off[0..n]; one CTA, chunked as compact_masks_kernel
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(const int* __restrict__ cnt, int n, int* __restrict__ off) {
    __shared__ int warp_tot[32];
    __shared__ int carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < n ? cnt[i] : 0;
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_tot[warp] = x;
        __syncthreads();
        int w_off = carry;
        for (int w = 0; w < warp; ++w) w_off += warp_tot[w];
        if (i < n) off[i] = w_off + x - v;
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int w = 0; w < 32; ++w) t += warp_tot[w];
            carry += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) off[n] = carry;
}

// bucket fill (arbitrary order inside a bucket), then every entry's rank inside its bucket = the number of smaller entry ids
__global__ void __launch_bounds__(256) patch_rows_fill_kernel(PatchRows pr, const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                              const int* __restrict__ off, int* __restrict__ cur, int* __restrict__ keys) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 2 * pr.per_side) return;
    const int row = pr.row_of(e, R, Q);
    if (row >= 0) keys[off[row] + atomicAdd(&cur[row], 1)] = (int)e;
}

__global__ void __launch_bounds__(256) patch_rows_rank_kernel(PatchRows pr, const __grid_constant__ Segs R, const __grid_constant__ Segs Q,
                                                              const int* __restrict__ off, const int* __restrict__ keys,
                                                              int* __restrict__ sorted) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 2 * pr.per_side) return;
    const int row = pr.row_of(e, R, Q);
    if (row < 0) return;
    const int b = off[row], n = off[row + 1] - b;
    int rank = 0;
    for (int s = 0; s < n; ++s) rank += keys[b + s] < (int)e;
    sorted[b + rank] = (int)e;
}

// grad row r = sum over its entries, in entry order, of tmp[entry]; rows without entries get zeros.  One CTA per row.
__global__ void __launch_bounds__(128) patch_rows_reduce_kernel(const float* __restrict__ tmp, int C, const int* __restrict__ off,
                                                                const int* __restrict__ sorted, int n_ref_rows, float* __restrict__ gref,
                                                                float* __restrict__ gsrc) {
    const int row = blockIdx.x;
    float* out = row < n_ref_rows ? gref + (long long)row * C : gsrc + (long long)(row - n_ref_rows) * C;
    const int b = off[row], n = off[row + 1] - b;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < n; ++k) s += tmp[(long long)sorted[b + k] * C + c];
        out[c] = s;
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

size_t geob200_sinkhorn_backward_workspace_bytes(int64_t n_patches, int64_t k, int64_t num_iterations) {
    const size_t K1 = (size_t)k + 1;
    return align_up(4 * (size_t)n_patches * 2 * (size_t)num_iterations * K1, 256) + align_up(4 * (size_t)n_patches, 256) + 256;
}

int geob200_sinkhorn_backward(const float* scores, const uint8_t* row_masks, const uint8_t* col_masks, const float* alpha, int64_t n_patches,
                              int64_t k, int64_t num_iterations, float inf, const float* grad_out, float* grad_scores, float* grad_alpha,
                              void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_patches >= 0 && n_patches <= 0x7fffffff, "sinkhorn_backward: bad patch count");
    GEOB_REQUIRE(k == 32 || k == 64 || k == 128, "sinkhorn_backward: k must be 32, 64 or 128, got %lld", (long long)k);
    GEOB_REQUIRE(num_iterations >= 1 && num_iterations <= 100000, "sinkhorn_backward: num_iterations must be in 1..100000");
    GEOB_REQUIRE(inf > 0.f, "sinkhorn_backward: inf must be positive");
    GEOB_REQUIRE(scores != nullptr && row_masks != nullptr && col_masks != nullptr && alpha != nullptr && grad_out != nullptr &&
                     grad_scores != nullptr && grad_alpha != nullptr,
                 "sinkhorn_backward: null pointer");
    GEOB_REQUIRE(workspace_bytes >= geob200_sinkhorn_backward_workspace_bytes(n_patches, k, num_iterations),
                 "sinkhorn_backward: workspace too small");
    const int K1 = (int)k + 1, ld = K1 | 1;
    const size_t smem = sizeof(float) * (2 * (size_t)K1 * ld + 6 * K1) + 2 * (size_t)K1;
    Arena ar(workspace, workspace_bytes);
    float* hist = ar.take<float>((size_t)n_patches * 2 * num_iterations * K1);
    float* part = ar.take<float>((size_t)n_patches);
    GEOB_REQUIRE(ar.ok(), "sinkhorn_backward: workspace accounting error");
    int n_launch = 1;
    if (n_patches > 0) {
#define LAUNCH_SK_BWD(KV, LPRV, MT, MB)                                                                                               \
    {                                                                                                                                 \
        if (smem > 48 * 1024 && ensure_max_smem((const void*)sinkhorn_bwd_kernel<KV, LPRV, MT, MB>)) return -1;                       \
        sinkhorn_bwd_kernel<KV, LPRV, MT, MB><<<(unsigned)n_patches, MT, smem, st>>>(scores, row_masks, col_masks, alpha,                 \
                                                                                 (int)num_iterations, inf, grad_out, hist,            \
                                                                                 grad_scores, part);                                  \
    }
        if (k == 32) LAUNCH_SK_BWD(32, 8, 288, 2)             // two CTAs per SM where registers allow, one at K = 128
        else if (k == 64) LAUNCH_SK_BWD(64, 8, 544, 2)
        else LAUNCH_SK_BWD(128, 4, 544, 1)
#undef LAUNCH_SK_BWD
        n_launch += 1;
    }
    sum_partials_kernel<<<1, 256, 0, st>>>(part, (int)n_patches, grad_alpha);
    GEOB_CHECK_LAUNCH();
    count_launches(n_launch);
    return 0;
}

size_t geob200_patch_scores_backward_batched_workspace_bytes(int64_t n_rows, int64_t n_patches_total, int64_t k, int64_t channels) {
    const size_t e = 2 * (size_t)n_patches_total * (size_t)k, r = (size_t)n_rows;
    return align_up(4 * e * (size_t)channels, 256) + 2 * align_up(4 * e, 256) + 2 * align_up(4 * r, 256) + align_up(4 * (r + 1), 256) + 256;
}

int geob200_patch_scores_backward_batched(const float* ref_feats, const float* src_feats, int64_t channels, int64_t n_pairs,
                                          const int64_t* cloud_points, const int64_t* ref_knn_indices, const int64_t* src_knn_indices,
                                          int64_t n_patches, int64_t k, const float* grad_scores, float* grad_ref_feats,
                                          float* grad_src_feats, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "patch_scores_backward_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(k == 32 || k == 64 || k == 128, "patch_scores_backward_batched: num_points_in_patch=%lld unsupported (32, 64, 128)",
                 (long long)k);
    GEOB_REQUIRE(channels >= 1 && channels <= 65536, "patch_scores_backward_batched: 1..65536 channels");
    GEOB_REQUIRE(n_patches >= 0 && n_patches <= 65535, "patch_scores_backward_batched: 0..65535 patches per pair");
    GEOB_REQUIRE(grad_ref_feats != nullptr && grad_src_feats != nullptr, "patch_scores_backward_batched: null gradient pointer");
    Segs R, Q;
    if (segs_from_counts(&R, n_pairs, cloud_points) || segs_from_counts(&Q, n_pairs, cloud_points + n_pairs)) return -1;
    const int64_t n_ref = (int64_t)R.start[R.n - 1] + R.count[R.n - 1], n_src = (int64_t)Q.start[Q.n - 1] + Q.count[Q.n - 1];
    const int64_t rows = n_ref + n_src, P_all = n_pairs * n_patches, E = 2 * P_all * k;
    GEOB_REQUIRE(rows < (1ll << 31) - 1 && E < (1ll << 31), "patch_scores_backward_batched: too many rows or patch entries");
    GEOB_REQUIRE(E == 0 || (grad_scores != nullptr && ref_knn_indices != nullptr && src_knn_indices != nullptr),
                 "patch_scores_backward_batched: null pointer");
    GEOB_REQUIRE(workspace_bytes >= geob200_patch_scores_backward_batched_workspace_bytes(rows, P_all, k, channels),
                 "patch_scores_backward_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    float* tmp = ar.take<float>((size_t)E * channels);
    int* keys = ar.take<int>((size_t)E);
    int* sorted = ar.take<int>((size_t)E);
    int* cnt = ar.take<int>((size_t)rows);
    int* cur = ar.take<int>((size_t)rows);
    int* off = ar.take<int>((size_t)rows + 1);
    GEOB_REQUIRE(ar.ok(), "patch_scores_backward_batched: workspace accounting error");
    const size_t smem = sizeof(float) * ((size_t)k * (k + 1) + (size_t)k * 33);
    if (smem > 48 * 1024) {
        const void* fn = k == 128 ? (const void*)patch_scores_bwd_kernel<128> : k == 64 ? (const void*)patch_scores_bwd_kernel<64>
                                                                                        : (const void*)patch_scores_bwd_kernel<32>;
        if (ensure_max_smem(fn)) return -1;
    }
    if (rows == 0) return 0;
    int n_launch = 0;
    const PatchRows pr{(const long long*)ref_knn_indices, (const long long*)src_knn_indices, P_all * k, (int)k, (int)n_patches, (int)n_ref};
    if (E > 0) {
        const float div = sqrtf((float)channels);      // as the forward: feats_f.shape[1] ** 0.5
        const dim3 grid((unsigned)n_patches, (unsigned)n_pairs, 2);
#define LAUNCH_PSB(KV) patch_scores_bwd_kernel<KV><<<grid, 256, smem, st>>>(ref_feats, src_feats, R, Q, (int)channels,                  \
                                                                            (const long long*)ref_knn_indices,                          \
                                                                            (const long long*)src_knn_indices, div, grad_scores, tmp)
        if (k == 128) LAUNCH_PSB(128);
        else if (k == 64) LAUNCH_PSB(64);
        else LAUNCH_PSB(32);
#undef LAUNCH_PSB
        GEOB_CHECK_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int) * (size_t)rows, st));
        GEOB_CHECK_CUDA(cudaMemsetAsync(cur, 0, sizeof(int) * (size_t)rows, st));
        const unsigned ge = (unsigned)((E + 255) / 256);
        patch_rows_count_kernel<<<ge, 256, 0, st>>>(pr, R, Q, cnt);
        exclusive_scan_kernel<<<1, 1024, 0, st>>>(cnt, (int)rows, off);
        patch_rows_fill_kernel<<<ge, 256, 0, st>>>(pr, R, Q, off, cur, keys);
        patch_rows_rank_kernel<<<ge, 256, 0, st>>>(pr, R, Q, off, keys, sorted);
        n_launch += 5;
    } else {
        GEOB_CHECK_CUDA(cudaMemsetAsync(off, 0, sizeof(int) * ((size_t)rows + 1), st));
    }
    patch_rows_reduce_kernel<<<(unsigned)rows, 128, 0, st>>>(tmp, (int)channels, off, sorted, (int)n_ref, grad_ref_feats, grad_src_feats);
    GEOB_CHECK_LAUNCH();
    count_launches(n_launch + 1);
    return 0;
}

}  // extern "C"
