// Backward of the KPConv-FPN backbone ops (kpconv.cu): KPConv, Linear, GroupNorm (+ residual, + LeakyReLU), max-pool and
// nearest-upsample + concat.
//
// No float atomics: every reduction has a fixed order, so two backward runs give the same bits.
//   - Reductions over the rows (dW of KPConv and Linear, the bias gradients) run on fixed 256-row chunks, one partial per chunk,
//     folded in chunk order in double (atb_partial_kernel / atb_fold_kernel).
//   - Scatters into support rows (KPConv's d s_feats, max-pool, upsample) go through a CSR transpose of the index table built by a
//     counting sort: integer atomics place the entries, a rank pass orders each row's entries by entry id = (query row, column), and
//     one warp per support row sums them in that order.
//   - GroupNorm sums run per 128-row tile of one cloud (a tile never straddles a cloud, so a pair's sums never see another
//     pair's rows), one thread per channel walking the rows in order, then a fixed-order fold.
#include "common.cuh"
#include "geob200.h"
#include "kpconv.cuh"

namespace geob200 {

__global__ void __launch_bounds__(1024) exclusive_scan_kernel(const int* __restrict__ cnt, int n, int* __restrict__ off);   // matching.cu

// ---------------------------------------------------------------------------------------------------------- CSR transpose
// entry e = m * cols + h of a (rows, cols) index table with row stride ld; it refers to support row tbl[m][h] when that lies in
// [0, n_support), else (sentinel) to nothing
struct IndexTable {
    const long long* idx;
    long long ld;
    int rows, cols, n_support;
    __device__ __forceinline__ int target(int e) const {
        const int m = e / cols, h = e - m * cols;
        const long long v = idx[(long long)m * ld + h];
        return (v >= 0 && v < n_support) ? (int)v : -1;
    }
};

__global__ void __launch_bounds__(256) csr_count_kernel(IndexTable t, int* __restrict__ cnt) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.rows * t.cols) return;
    const int s = t.target(e);
    if (s >= 0) atomicAdd(&cnt[s], 1);
}

__global__ void __launch_bounds__(256) csr_fill_kernel(IndexTable t, const int* __restrict__ off, int* __restrict__ cur,
                                                       int* __restrict__ keys) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.rows * t.cols) return;
    const int s = t.target(e);
    if (s >= 0) keys[off[s] + atomicAdd(&cur[s], 1)] = e;
}

// every entry's rank inside its support row = the number of smaller entry ids there
__global__ void __launch_bounds__(256) csr_rank_kernel(IndexTable t, const int* __restrict__ off, const int* __restrict__ keys,
                                                       int* __restrict__ sorted) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.rows * t.cols) return;
    const int s = t.target(e);
    if (s < 0) return;
    const int b = off[s], n = off[s + 1] - b;
    int rank = 0;
    for (int i = 0; i < n; ++i) rank += keys[b + i] < e;
    sorted[b + rank] = e;
}

struct Csr { int* off; int* sorted; };

static size_t csr_bytes(int64_t entries, int64_t n_support) {
    return 3 * align_up((size_t)(n_support + 1) * 4, 256) + 2 * align_up((size_t)entries * 4, 256);
}

static int build_csr(const IndexTable& t, Arena& ar, Csr* out, cudaStream_t st) {
    const int ns = t.n_support, ne = t.rows * t.cols;
    int* cnt = ar.take<int>(ns + 1);
    int* cur = ar.take<int>(ns + 1);
    out->off = ar.take<int>(ns + 1);
    int* keys = ar.take<int>(ne);
    out->sorted = ar.take<int>(ne);
    GEOB_CHECK_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int) * (ns + 1), st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(cur, 0, sizeof(int) * (ns + 1), st));
    const unsigned g = (unsigned)((ne + 255) / 256);
    csr_count_kernel<<<g, 256, 0, st>>>(t, cnt);
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(cnt, ns, out->off);
    csr_fill_kernel<<<g, 256, 0, st>>>(t, out->off, cur, keys);
    csr_rank_kernel<<<g, 256, 0, st>>>(t, out->off, keys, out->sorted);
    count_launches(4);
    return 0;
}

// ---------------------------------------------------------------------------------------------------------- C = A^T (s . B)
// C[i][j] = sum_m A[m][i] * (B[m][j] * s[m]) for i < ka, j < n; A == nullptr stands for a column of ones (ka = 1: column sums),
// s == nullptr for ones.  fp32 FMAs over a 256-row chunk per CTA (blockIdx.z), 64 x 64 output tile, 4 x 4 per thread; the chunk
// partials are folded in chunk order in double.  The same reduction serves KPConv's dW (A = gathered features, B = dOut,
// s = 1 / n_valid), Linear's dW (A = dY, B = X) and every bias gradient.
constexpr int ATB_ROWS = 256;
constexpr int ATB_T = 64;

__global__ void __launch_bounds__(256) atb_partial_kernel(const float* __restrict__ A, long long lda, const float* __restrict__ B,
                                                          long long ldb, const float* __restrict__ s, int M, int ka, int n,
                                                          float* __restrict__ part) {
    __shared__ float As[16][ATB_T];
    __shared__ float Bs[16][ATB_T];
    const int i0 = blockIdx.y * ATB_T, j0 = blockIdx.x * ATB_T;
    const int r0 = blockIdx.z * ATB_ROWS, r1 = min(M, r0 + ATB_ROWS);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
    for (int m0 = r0; m0 < r1; m0 += 16) {
        for (int e = threadIdx.x; e < 16 * ATB_T; e += 256) {
            const int r = e / ATB_T, c = e % ATB_T;
            const int m = m0 + r;
            const bool row_ok = m < r1;
            float av = 0.f, bv = 0.f;
            if (row_ok && i0 + c < ka) av = A != nullptr ? A[(long long)m * lda + i0 + c] : 1.f;
            if (row_ok && j0 + c < n) {
                bv = B[(long long)m * ldb + j0 + c];
                if (s != nullptr) bv *= s[m];
            }
            As[r][c] = av;
            Bs[r][c] = bv;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            float a[4], b[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { a[u] = As[r][ty + 16 * u]; b[u] = Bs[r][tx + 16 * u]; }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
        }
        __syncthreads();
    }
    float* out = part + (long long)blockIdx.z * ka * n;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int i = i0 + ty + 16 * u;
        if (i >= ka) continue;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int j = j0 + tx + 16 * v;
            if (j < n) out[(long long)i * n + j] = acc[u][v];
        }
    }
}

__global__ void __launch_bounds__(256) atb_fold_kernel(const float* __restrict__ part, int chunks, long long total, float* __restrict__ C) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    double s = 0.0;
    for (int z = 0; z < chunks; ++z) s += (double)part[(long long)z * total + i];
    C[i] = (float)s;
}

size_t atb_bytes(int64_t M, int64_t ka, int64_t n) {
    const int64_t chunks = (M + ATB_ROWS - 1) / ATB_ROWS;
    return chunks > 1 ? align_up((size_t)chunks * ka * n * 4, 256) : 0;
}

void atb(const float* A, long long lda, const float* B, long long ldb, const float* s, int64_t M, int64_t ka, int64_t n, float* C,
         float* part, cudaStream_t st) {
    const int chunks = (int)((M + ATB_ROWS - 1) / ATB_ROWS);
    const dim3 grid((unsigned)((n + ATB_T - 1) / ATB_T), (unsigned)((ka + ATB_T - 1) / ATB_T), (unsigned)chunks);
    if (chunks == 1) {
        atb_partial_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, s, (int)M, (int)ka, (int)n, C);
        count_launches(1);
        return;
    }
    atb_partial_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, s, (int)M, (int)ka, (int)n, part);
    const long long total = ka * n;
    atb_fold_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(part, chunks, total, C);
    count_launches(2);
}

__global__ void __launch_bounds__(256) relu_grad_kernel(const float* __restrict__ dy, const float* __restrict__ y, long long total,
                                                        float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) out[i] = y[i] > 0.f ? dy[i] : 0.f;
}

// ---------------------------------------------------------------------------------------------------------- KPConv
// c_in = 1 (first layer): wf[m][k] = sum_h influence[m][h][k] * f[nbr[m][h]] and inv_count[m], as kpconv_c1_kernel forms them
// (half a warp per query, the same 16-lane shuffle tree)
__global__ void __launch_bounds__(256) kpconv_c1_wf_kernel(const float* __restrict__ feats, const float* __restrict__ q_pts,
                                                           const float* __restrict__ s_pts, const long long* __restrict__ nbr, int H,
                                                           const float* __restrict__ kp, float sigma, int Ns, int M,
                                                           float* __restrict__ wf, float* __restrict__ inv_count) {
    __shared__ float kp_s[KP * 3];
    if (threadIdx.x < KP * 3) kp_s[threadIdx.x] = kp[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sl = lane & 15;
    const int m = blockIdx.x * 16 + warp * 2 + (lane >> 4);
    const bool live = m < M;
    float acc[KP];
#pragma unroll
    for (int k = 0; k < KP; ++k) acc[k] = 0.f;
    int npos = 0;
    if (live) {
        const float qx = q_pts[3ll * m], qy = q_pts[3ll * m + 1], qz = q_pts[3ll * m + 2];
        for (int h = sl; h < H; h += 16) {
            const long long idx = nbr[(long long)m * H + h];
            if (idx >= 0 && idx < Ns) {
                float w[KP];
                influence15(kp_s, s_pts[3 * idx] - qx, s_pts[3 * idx + 1] - qy, s_pts[3 * idx + 2] - qz, 0.f, sigma, w);
                const float f = feats[idx];
                npos += (f > 0.f);
#pragma unroll
                for (int k = 0; k < KP; ++k) acc[k] = fmaf(w[k], f, acc[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < KP; ++k) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) npos += __shfl_xor_sync(0xffffffffu, npos, o);
    if (live && sl == 0) {
#pragma unroll
        for (int k = 0; k < KP; ++k) wf[(long long)m * KP + k] = acc[k];
        inv_count[m] = 1.0f / (float)max(npos, 1);
    }
}

// d s_feats[s][c] = sum over the entries (m, h) of support row s, in entry order, of inv_count[m] * sum_k influence[m][h][k] *
// dwf[m][k c_in + c].  One warp per support row, lanes over 4 channel groups of 32 (c_in = 1: lane 0 alone); the influences are
// recomputed with the forward's arithmetic.  Rows no query references get zeros.
__global__ void __launch_bounds__(256) kpconv_dx_kernel(const float* __restrict__ dwf, const float* __restrict__ inv_count,
                                                        const float* __restrict__ q_pts, const float* __restrict__ s_pts,
                                                        const float* __restrict__ kp, float sigma, int H, int Ns, int Cin,
                                                        const int* __restrict__ off, const int* __restrict__ sorted,
                                                        float* __restrict__ dx) {
    __shared__ float kp_s[KP * 3];
    if (threadIdx.x < KP * 3) kp_s[threadIdx.x] = kp[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (s >= Ns) return;
    const int b = off[s], ne = off[s + 1] - b;
    const float sx = s_pts[3ll * s], sy = s_pts[3ll * s + 1], sz = s_pts[3ll * s + 2];
    for (int c0 = 0; c0 < Cin; c0 += 128) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int i = 0; i < ne; ++i) {
            const int m = sorted[b + i] / H;
            float w[KP];
            influence15(kp_s, sx - q_pts[3ll * m], sy - q_pts[3ll * m + 1], sz - q_pts[3ll * m + 2], 0.f, sigma, w);
            const float sc = inv_count[m];
            const float* row = dwf + (long long)m * KP * Cin + c0 + lane;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (c0 + 32 * u + lane < Cin) {
                    float t = 0.f;
#pragma unroll
                    for (int k = 0; k < KP; ++k) t = fmaf(w[k], row[(long long)k * Cin + 32 * u], t);
                    acc[u] = fmaf(sc, t, acc[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (c0 + 32 * u + lane < Cin) dx[(long long)s * Cin + c0 + 32 * u + lane] = acc[u];
    }
}

// ---------------------------------------------------------------------------------------------------------- GroupNorm
// 128-row tiles inside the clouds: tile t of cloud c covers rows start[c] + 128 (t - base[c]) ...; every CTA derives the bases
struct TileOf { int cloud, r0, r1; };

__device__ __forceinline__ TileOf tile_of(const GnSeg& seg, int tile) {
    int base = 0;
    for (int c = 0; c < seg.n_clouds; ++c) {
        const int rows = seg.start[c + 1] - seg.start[c];
        const int nt = (rows + 127) / 128;
        if (tile < base + nt) {
            const int r0 = seg.start[c] + 128 * (tile - base);
            return {c, r0, min(seg.start[c + 1], r0 + 128)};
        }
        base += nt;
    }
    return {-1, 0, 0};
}

static int seg_tiles(const GnSeg& seg) {
    int n = 0;
    for (int c = 0; c < seg.n_clouds; ++c) n += (seg.start[c + 1] - seg.start[c] + 127) / 128;
    return n;
}

// per tile and channel: (sum x, sum x^2) in double, rows in order
__global__ void __launch_bounds__(256) gnb_stats_tile_kernel(const float* __restrict__ x, int C, GnSeg seg, double2* __restrict__ part) {
    const TileOf t = tile_of(seg, blockIdx.x);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double s = 0.0, s2 = 0.0;
        for (int r = t.r0; r < t.r1; ++r) {
            const double v = (double)x[(long long)r * C + c];
            s += v;
            s2 += v * v;
        }
        part[(long long)blockIdx.x * C + c] = make_double2(s, s2);
    }
}

// one 128-thread CTA per (group, pair): fold the (tile, channel) partials of the pair's tiles with a fixed assignment and tree, then
// mean / rstd with the forward's formula (gn_seg_finalize_kernel), kept in double
__global__ void __launch_bounds__(128) gnb_stats_fold_kernel(const double2* __restrict__ part, int C, int G, double eps, GnSeg seg,
                                                             double2* __restrict__ mean_rstd) {
    __shared__ double red[8];
    __shared__ int tb[GEOB_MAX_CLOUDS + 1];
    const int g = blockIdx.x, p = blockIdx.y, cpg = C / G;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        tb[0] = 0;
        for (int c = 0; c < seg.n_clouds; ++c) tb[c + 1] = tb[c] + (seg.start[c + 1] - seg.start[c] + 127) / 128;
    }
    __syncthreads();
    double sa = 0.0, sb = 0.0;
    long long rows = 0;
    for (int c = p; c < seg.n_clouds; c += seg.n_pairs) {
        rows += seg.start[c + 1] - seg.start[c];
        const int n = (tb[c + 1] - tb[c]) * cpg;
        for (int i = threadIdx.x; i < n; i += 128) {
            const double2 v = part[(long long)(tb[c] + i / cpg) * C + g * cpg + i % cpg];
            sa += v.x;
            sb += v.y;
        }
    }
    sa = warp_sum_d(sa);
    sb = warp_sum_d(sb);
    if (lane == 0) { red[2 * warp] = sa; red[2 * warp + 1] = sb; }
    __syncthreads();
    if (threadIdx.x == 0) {
        sa = (red[0] + red[2]) + (red[4] + red[6]);
        sb = (red[1] + red[3]) + (red[5] + red[7]);
        double mean = 0.0, rstd = 0.0;
        if (rows > 0) {
            const double count = (double)cpg * (double)rows;
            mean = sa / count;
            double var = sb / count - mean * mean;
            if (var < 0.0) var = 0.0;
            rstd = 1.0 / sqrt(var + eps);
        }
        mean_rstd[(long long)p * G + g] = make_double2(mean, rstd);
    }
}

// gradient at the normalised value + beta (+ residual): the upstream gradient through the LeakyReLU, whose derivative follows the
// sign of the pre-activation as torch's does (slope at 0).  With slope >= 0 the output y has that sign, so y decides.
__device__ __forceinline__ float gn_dz(const float* __restrict__ dy, const float* __restrict__ y, long long i, int leaky, float slope) {
    const float d = dy[i];
    return (leaky && !(y[i] > 0.f)) ? d * slope : d;
}

// per tile and channel: (sum dz, sum dz * xhat) in double; writes the residual's gradient (= dz) on the way
__global__ void __launch_bounds__(256) gnb_grad_tile_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                            const float* __restrict__ dy, const double2* __restrict__ mean_rstd, int C,
                                                            int G, int leaky, float slope, GnSeg seg, double2* __restrict__ part,
                                                            float* __restrict__ dres) {
    const TileOf t = tile_of(seg, blockIdx.x);
    const int p = t.cloud % seg.n_pairs, cpg = C / G;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const double2 mr = mean_rstd[(long long)p * G + c / cpg];
        double s = 0.0, s2 = 0.0;
        for (int r = t.r0; r < t.r1; ++r) {
            const long long i = (long long)r * C + c;
            const float dz = gn_dz(dy, y, i, leaky, slope);
            const double xh = ((double)x[i] - mr.x) * mr.y;
            s += (double)dz;
            s2 += (double)dz * xh;
            if (dres != nullptr) dres[i] = dz;
        }
        part[(long long)blockIdx.x * C + c] = make_double2(s, s2);
    }
}

// One CTA: per (pair, channel) the tile sums in tile order -> S[p][c]; dbeta[c] / dgamma[c] = sums over the pairs in pair order;
// coef[p][g] = (sum_{c in g} gamma_c S1[p][c], sum gamma_c S2[p][c]) / (cpg * rows of pair p)
__global__ void __launch_bounds__(1024) gnb_fold_kernel(const double2* __restrict__ part, const float* __restrict__ gamma, int C, int G,
                                                        GnSeg seg, double2* __restrict__ S, float* __restrict__ dgamma,
                                                        float* __restrict__ dbeta, double2* __restrict__ coef) {
    __shared__ int tb[GEOB_MAX_CLOUDS + 1];
    if (threadIdx.x == 0) {
        tb[0] = 0;
        for (int c = 0; c < seg.n_clouds; ++c) tb[c + 1] = tb[c] + (seg.start[c + 1] - seg.start[c] + 127) / 128;
    }
    __syncthreads();
    const int P = seg.n_pairs, cpg = C / G;
    for (int i = threadIdx.x; i < P * C; i += blockDim.x) {
        const int p = i / C, c = i % C;
        double a = 0.0, b = 0.0;
        for (int cl = p; cl < seg.n_clouds; cl += P)
            for (int t = tb[cl]; t < tb[cl + 1]; ++t) {
                const double2 v = part[(long long)t * C + c];
                a += v.x;
                b += v.y;
            }
        S[i] = make_double2(a, b);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double a = 0.0, b = 0.0;
        for (int p = 0; p < P; ++p) { a += S[(long long)p * C + c].x; b += S[(long long)p * C + c].y; }
        if (dbeta != nullptr) dbeta[c] = (float)a;
        if (dgamma != nullptr) dgamma[c] = (float)b;
    }
    for (int i = threadIdx.x; i < P * G; i += blockDim.x) {
        const int p = i / G, g = i % G;
        long long rows = 0;
        for (int cl = p; cl < seg.n_clouds; cl += P) rows += seg.start[cl + 1] - seg.start[cl];
        double a = 0.0, b = 0.0;
        for (int j = 0; j < cpg; ++j) {
            const double gm = (double)gamma[g * cpg + j];
            a += gm * S[(long long)p * C + g * cpg + j].x;
            b += gm * S[(long long)p * C + g * cpg + j].y;
        }
        const double cnt = rows > 0 ? (double)cpg * (double)rows : 1.0;
        coef[i] = make_double2(a / cnt, b / cnt);
    }
}

// dx = rstd * (gamma dz - mean_g(gamma dz) - xhat mean_g(gamma dz xhat)) with the statistics of the row's pair
__global__ void __launch_bounds__(256) gnb_apply_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                                        const double2* __restrict__ mean_rstd, const float* __restrict__ gamma,
                                                        const double2* __restrict__ coef, long long total, int C, int G, int leaky,
                                                        float slope, GnSeg seg, float* __restrict__ dx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int r = (int)(i / C), c = (int)(i % C);
    const int p = cloud_of(seg.start, seg.n_clouds, r) % seg.n_pairs, g = c / (C / G);
    const double2 mr = mean_rstd[(long long)p * G + g];
    const double2 k = coef[(long long)p * G + g];
    const double xh = ((double)x[i] - mr.x) * mr.y;
    const double dxh = (double)gamma[c] * (double)gn_dz(dy, y, i, leaky, slope);
    dx[i] = (float)(mr.y * (dxh - k.x - xh * k.y));
}

// ---------------------------------------------------------------------------------------------------------- max-pool
// arg[m][c] = the first column of row m's neighbours (within the pair's width) holding the maximum, -1 when the zero shadow row wins
__global__ void __launch_bounds__(256) maxpool_arg_kernel(const float* __restrict__ x, const long long* __restrict__ nbr, int H, int Ns,
                                                          int M, int C, GnSeg seg, const int* __restrict__ cloud_max,
                                                          int* __restrict__ arg) {
    __shared__ int width[GEOB_MAX_CLOUDS];
    for (int i = threadIdx.x; i < seg.n_clouds; i += blockDim.x) {
        int w = H;
        if (cloud_max != nullptr) {
            w = 0;
            for (int c = i % seg.n_pairs; c < seg.n_clouds; c += seg.n_pairs) w = max(w, cloud_max[c]);
            w = min(H, w);
        }
        width[i] = w;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int m = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (m >= M) return;
    const int W = width[cloud_of(seg.start, seg.n_clouds, m)];
    const long long* row = nbr + (long long)m * H;
    for (int c = lane; c < C; c += 32) {
        float best = -INFINITY;
        int a = -1;
        for (int h = 0; h < W; ++h) {
            const long long idx = row[h];
            const bool real = idx >= 0 && idx < Ns;
            const float v = real ? x[idx * C + c] : 0.f;
            if (v > best) { best = v; a = real ? h : -1; }
        }
        arg[(long long)m * C + c] = a;
    }
}

// dx[s][c] = sum over the entries (m, h) of support row s, in entry order, of dy[m][c] where column h won channel c of row m
__global__ void __launch_bounds__(256) maxpool_scatter_kernel(const float* __restrict__ dy, const int* __restrict__ arg, int H, int Ns, int C,
                                                              const int* __restrict__ off, const int* __restrict__ sorted,
                                                              float* __restrict__ dx) {
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (s >= Ns) return;
    const int b = off[s], ne = off[s + 1] - b;
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
        for (int i = 0; i < ne; ++i) {
            const int e = sorted[b + i], m = e / H, h = e - m * H;
            if (arg[(long long)m * C + c] == h) acc += dy[(long long)m * C + c];
        }
        dx[(long long)s * C + c] = acc;
    }
}

// ---------------------------------------------------------------------------------------------------------- upsample + concat
// dx[s][c] = sum over the fine rows m with up[m][0] = s, in row order, of dy[m][c] (c < c1)
__global__ void __launch_bounds__(256) upsample_scatter_kernel(const float* __restrict__ dy, int ldy, int Ns, int C1,
                                                               const int* __restrict__ off, const int* __restrict__ sorted,
                                                               float* __restrict__ dx) {
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (s >= Ns) return;
    const int b = off[s], ne = off[s + 1] - b;
    for (int c = lane; c < C1; c += 32) {
        float acc = 0.f;
        for (int i = 0; i < ne; ++i) acc += dy[(long long)sorted[b + i] * ldy + c];
        dx[(long long)s * C1 + c] = acc;
    }
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_kpconv_backward_workspace_bytes(int64_t n_query, int64_t n_support, int64_t n_neighbors, int64_t c_in, int64_t c_out) {
    const int64_t ka = KP * c_in;
    return align_up((size_t)n_support, 256) + align_up((size_t)n_query * 4, 256) + align_up((size_t)n_query * ka * 4, 256) +
           atb_bytes(n_query, ka, c_out) + atb_bytes(n_query, 1, c_out) + csr_bytes(n_query * n_neighbors, n_support) + 1024;
}

int geob200_kpconv_backward(const float* s_feats, const float* q_points, const float* s_points, const int64_t* neighbors, int64_t n_query,
                            int64_t n_support, int64_t n_neighbors, const float* kernel_points, int64_t n_kernel, const float* weights,
                            int64_t c_in, int64_t c_out, float sigma, const float* grad_out, float* grad_feats, float* grad_weights,
                            float* grad_bias, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_kernel == KP, "kpconv_backward: kernel_size %lld unsupported", (long long)n_kernel);
    GEOB_REQUIRE(n_query > 0 && n_support > 0 && n_neighbors > 0 && c_out > 0, "kpconv_backward: empty input");
    GEOB_REQUIRE(c_in == 1 || c_in % 32 == 0, "kpconv_backward: c_in %lld must be 1 or a multiple of 32", (long long)c_in);
    GEOB_REQUIRE(n_query * n_neighbors < (1ll << 31) && n_query * KP * c_in < (1ll << 40), "kpconv_backward: neighbour table too large");
    GEOB_REQUIRE(s_feats != nullptr && q_points != nullptr && s_points != nullptr && neighbors != nullptr && kernel_points != nullptr &&
                 grad_out != nullptr && (grad_feats == nullptr || weights != nullptr), "kpconv_backward: null input");
    GEOB_REQUIRE(workspace != nullptr &&
                 workspace_bytes >= geob200_kpconv_backward_workspace_bytes(n_query, n_support, n_neighbors, c_in, c_out),
                 "kpconv_backward: workspace too small");
    const int64_t ka = KP * c_in;
    Arena ar(workspace, workspace_bytes);
    unsigned char* pos = ar.take<unsigned char>(n_support);
    float* inv_count = ar.take<float>(n_query);
    float* wf = ar.take<float>((size_t)n_query * ka);
    float* part = ar.take<float>(atb_bytes(n_query, ka, c_out) / 4 + atb_bytes(n_query, 1, c_out) / 4 + 1);
    const long long* nbr = (const long long*)neighbors;
    if (grad_bias != nullptr) atb(nullptr, 0, grad_out, c_out, nullptr, n_query, 1, c_out, grad_bias, part, st);
    if (grad_weights != nullptr || grad_feats != nullptr) {
        if (c_in == 1) {
            kpconv_c1_wf_kernel<<<(unsigned)((n_query + 15) / 16), 256, 0, st>>>(s_feats, q_points, s_points, nbr, (int)n_neighbors,
                                                                                 kernel_points, sigma, (int)n_support, (int)n_query, wf,
                                                                                 inv_count);
            count_launches(1);
        } else {
            kpconv_gather(s_feats, q_points, s_points, nbr, (int)n_neighbors, kernel_points, sigma, (int)n_support, (int)n_query, (int)c_in,
                          pos, wf, inv_count, st);
        }
    }
    // dW = wf^T (dOut / n_valid): (15 c_in, c_out), the layout of the weights
    if (grad_weights != nullptr) atb(wf, ka, grad_out, c_out, inv_count, n_query, ka, c_out, grad_weights, part, st);
    if (grad_feats != nullptr) {
        // dwf = dOut . W_flat^T (the 1 / n_valid scale is applied per query in kpconv_dx_kernel); overwrites wf
        const int rc = linear_img(grad_out, c_out, weights, nullptr, nullptr, wf, ka, n_query, ka, c_out, 0, stream);
        if (rc != 0) return rc;
        Csr csr;
        const IndexTable t{nbr, n_neighbors, (int)n_query, (int)n_neighbors, (int)n_support};
        if (build_csr(t, ar, &csr, st)) return -1;
        kpconv_dx_kernel<<<(unsigned)((n_support + 7) / 8), 256, 0, st>>>(wf, inv_count, q_points, s_points, kernel_points, sigma,
                                                                          (int)n_neighbors, (int)n_support, (int)c_in, csr.off,
                                                                          csr.sorted, grad_feats);
        count_launches(1);
    }
    GEOB_REQUIRE(ar.ok(), "kpconv_backward: workspace accounting error");
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_linear_backward_workspace_bytes(int64_t m, int64_t n, int64_t k, int relu) {
    return atb_bytes(m, n, k) + atb_bytes(m, 1, n) + (relu ? align_up((size_t)m * n * 4, 256) : 0) + 1024;
}

int geob200_linear_backward(const float* x, int64_t ldx, const float* weight_t, const float* relu_y, int64_t m, int64_t n, int64_t k,
                            const float* grad_y, float* grad_x, float* grad_weight, float* grad_bias, void* workspace, size_t workspace_bytes,
                            void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(m > 0 && n > 0 && k > 0, "linear_backward: empty problem");
    GEOB_REQUIRE(ldx >= k, "linear_backward: ldx %lld < k %lld", (long long)ldx, (long long)k);
    GEOB_REQUIRE(grad_y != nullptr && (grad_x == nullptr || weight_t != nullptr) && (grad_weight == nullptr || x != nullptr),
                 "linear_backward: null input");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_linear_backward_workspace_bytes(m, n, k, relu_y != nullptr),
                 "linear_backward: workspace too small");
    Arena ar(workspace, workspace_bytes);
    if (relu_y != nullptr) {                  // y = relu(x W^T + b): the gradient passes where the output is positive
        float* masked = ar.take<float>((size_t)m * n);
        const long long total = m * n;
        relu_grad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(grad_y, relu_y, total, masked);
        count_launches(1);
        grad_y = masked;
    }
    float* part = ar.take<float>(atb_bytes(m, n, k) / 4 + atb_bytes(m, 1, n) / 4 + 1);
    GEOB_REQUIRE(ar.ok(), "linear_backward: workspace accounting error");
    if (grad_bias != nullptr) atb(nullptr, 0, grad_y, n, nullptr, m, 1, n, grad_bias, part, st);
    if (grad_weight != nullptr) atb(grad_y, n, x, ldx, nullptr, m, n, k, grad_weight, part, st);   // dW = dY^T X  (n, k)
    if (grad_x != nullptr) {                                                                        // dX = dY W   (m, k)
        const int rc = linear_img(grad_y, n, weight_t, nullptr, nullptr, grad_x, k, m, k, n, 0, stream);
        if (rc != 0) return rc;
    }
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_group_norm_backward_batched_workspace_bytes(int64_t n_rows, int64_t channels, int64_t groups, int64_t n_pairs) {
    const size_t tiles = (size_t)(n_rows / 128 + 2 * n_pairs + 1);
    return 2 * align_up(tiles * channels * 16, 256) + align_up((size_t)n_pairs * channels * 16, 256) +
           2 * align_up((size_t)n_pairs * groups * 16, 256) + 1024;
}

int geob200_group_norm_backward_batched(const float* x, const float* y, int64_t n_rows, int64_t channels, int64_t groups, const float* gamma,
                                        float eps, int leaky, float slope, const float* grad_y, float* grad_x, float* grad_gamma,
                                        float* grad_beta, float* grad_residual, void* workspace, size_t workspace_bytes, void* stream,
                                        int64_t n_pairs, const int64_t* cloud_rows_h) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_rows > 0 && channels > 0 && groups > 0 && channels % groups == 0, "group_norm_backward: bad shape");
    GEOB_REQUIRE(x != nullptr && gamma != nullptr && grad_y != nullptr && grad_x != nullptr && (!leaky || y != nullptr),
                 "group_norm_backward: null input (y is needed with the LeakyReLU)");
    GEOB_REQUIRE(!leaky || slope >= 0.f, "group_norm_backward: negative LeakyReLU slope unsupported");
    GnSeg seg;
    if (make_seg(&seg, n_pairs, cloud_rows_h, n_rows, "group_norm_backward")) return -2;
    GEOB_REQUIRE(workspace != nullptr &&
                 workspace_bytes >= geob200_group_norm_backward_batched_workspace_bytes(n_rows, channels, groups, n_pairs),
                 "group_norm_backward: workspace too small");
    const int tiles = seg_tiles(seg);
    Arena ar(workspace, workspace_bytes);
    double2* part1 = ar.take<double2>((size_t)tiles * channels);
    double2* part2 = ar.take<double2>((size_t)tiles * channels);
    double2* S = ar.take<double2>((size_t)n_pairs * channels);
    double2* coef = ar.take<double2>((size_t)n_pairs * groups);
    double2* mean_rstd = ar.take<double2>((size_t)n_pairs * groups);
    GEOB_REQUIRE(ar.ok(), "group_norm_backward: workspace accounting error");
    const int C = (int)channels, G = (int)groups;
    gnb_stats_tile_kernel<<<tiles, 256, 0, st>>>(x, C, seg, part1);
    gnb_stats_fold_kernel<<<dim3(G, (unsigned)n_pairs), 128, 0, st>>>(part1, C, G, (double)eps, seg, mean_rstd);
    gnb_grad_tile_kernel<<<tiles, 256, 0, st>>>(x, y, grad_y, mean_rstd, C, G, leaky, slope, seg, part2, grad_residual);
    gnb_fold_kernel<<<1, 1024, 0, st>>>(part2, gamma, C, G, seg, S, grad_gamma, grad_beta, coef);
    const long long total = n_rows * channels;
    gnb_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, y, grad_y, mean_rstd, gamma, coef, total, C, G, leaky, slope, seg,
                                                                      grad_x);
    count_launches(5);
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_maxpool_backward_batched_workspace_bytes(int64_t n_query, int64_t n_support, int64_t n_neighbors, int64_t channels) {
    return align_up((size_t)n_query * channels * 4, 256) + csr_bytes(n_query * n_neighbors, n_support) + 1024;
}

int geob200_maxpool_backward_batched(const float* x, const int64_t* neighbors, int64_t n_query, int64_t n_support, int64_t n_neighbors,
                                     int64_t channels, const int32_t* cloud_max, int64_t n_pairs, const int64_t* cloud_rows_h,
                                     const float* grad_y, float* grad_x, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_query > 0 && n_support > 0 && n_neighbors > 0 && channels > 0, "maxpool_backward: empty input");
    GEOB_REQUIRE(n_query * n_neighbors < (1ll << 31), "maxpool_backward: neighbour table too large");
    GEOB_REQUIRE(x != nullptr && neighbors != nullptr && grad_y != nullptr && grad_x != nullptr, "maxpool_backward: null input");
    GnSeg seg;
    if (make_seg(&seg, n_pairs, cloud_rows_h, n_query, "maxpool_backward")) return -2;
    GEOB_REQUIRE(workspace != nullptr &&
                 workspace_bytes >= geob200_maxpool_backward_batched_workspace_bytes(n_query, n_support, n_neighbors, channels),
                 "maxpool_backward: workspace too small");
    Arena ar(workspace, workspace_bytes);
    int* arg = ar.take<int>((size_t)n_query * channels);
    const long long* nbr = (const long long*)neighbors;
    maxpool_arg_kernel<<<(unsigned)((n_query + 7) / 8), 256, 0, st>>>(x, nbr, (int)n_neighbors, (int)n_support, (int)n_query, (int)channels,
                                                                      seg, cloud_max, arg);
    count_launches(1);
    Csr csr;
    const IndexTable t{nbr, n_neighbors, (int)n_query, (int)n_neighbors, (int)n_support};
    if (build_csr(t, ar, &csr, st)) return -1;
    GEOB_REQUIRE(ar.ok(), "maxpool_backward: workspace accounting error");
    maxpool_scatter_kernel<<<(unsigned)((n_support + 7) / 8), 256, 0, st>>>(grad_y, arg, (int)n_neighbors, (int)n_support, (int)channels,
                                                                            csr.off, csr.sorted, grad_x);
    count_launches(1);
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_upsample_concat_backward_workspace_bytes(int64_t n_query, int64_t n_support) { return csr_bytes(n_query, n_support) + 1024; }

int geob200_upsample_concat_backward(const int64_t* up_indices, int64_t up_stride, int64_t n_query, int64_t n_support, int64_t c1, int64_t c2,
                                     const float* grad_y, float* grad_x, float* grad_skip, void* workspace, size_t workspace_bytes,
                                     void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_query > 0 && n_support > 0 && c1 > 0 && c2 >= 0 && up_stride >= 1, "upsample_concat_backward: bad shape");
    GEOB_REQUIRE(up_indices != nullptr && grad_y != nullptr && grad_x != nullptr && (grad_skip == nullptr || c2 > 0),
                 "upsample_concat_backward: null input");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_upsample_concat_backward_workspace_bytes(n_query, n_support),
                 "upsample_concat_backward: workspace too small");
    Arena ar(workspace, workspace_bytes);
    Csr csr;
    const IndexTable t{(const long long*)up_indices, up_stride, (int)n_query, 1, (int)n_support};
    if (build_csr(t, ar, &csr, st)) return -1;
    GEOB_REQUIRE(ar.ok(), "upsample_concat_backward: workspace accounting error");
    upsample_scatter_kernel<<<(unsigned)((n_support + 7) / 8), 256, 0, st>>>(grad_y, (int)(c1 + c2), (int)n_support, (int)c1, csr.off,
                                                                             csr.sorted, grad_x);
    count_launches(1);
    if (grad_skip != nullptr)
        GEOB_CHECK_CUDA(cudaMemcpy2DAsync(grad_skip, c2 * 4, grad_y + c1, (c1 + c2) * 4, c2 * 4, n_query, cudaMemcpyDeviceToDevice, st));
    GEOB_CHECK_LAUNCH();
    return 0;
}

}  // extern "C"
