// Backward of the geometric transformer ops (attention.cu, attention_tma.cu, gse_table.cu): residual LayerNorm, row
// L2-normalisation, head_project (proj_p moved onto q), multi-head attention with and without the structure term, and the
// structure embedding E = proj_d(s(d)) + max_k proj_a(s(a_k)).
//
// No float atomics: every reduction has a fixed order, so two backward runs give the same bits.
//   - Sums over rows (dgamma, dbeta, dWp, dbp, the embedding biases) use the row-chunk reduction of kpconv_grad.cu (atb): fp32
//     partials per 256-row chunk, folded in chunk order in double.
//   - The attention products (dP = dO v^T, dV = P^T dO, dQ = dS' K, dK = dS'^T Q) are register-tiled CUDA-core GEMMs: one thread
//     owns each output element and walks the contraction in order.
//   - The E pass streams E[n] once per query row n: every warp takes a fixed set of keys, the warps' dqp partials are folded in warp
//     order through shared memory.
//   - The embedding weight gradients are fp32 sums over 2048-row chunks (one CTA per 64 x 64 tile and chunk), folded in chunk order
//     in double.
#include "common.cuh"
#include "geob200.h"
#include "gse_table.cuh"
#include "kpconv.cuh"

namespace geob200 {

// ---------------------------------------------------------------------------------------------------------- LayerNorm
// y = LN(a + b) gamma + beta: one warp per row, x = a + b and its statistics recomputed with the forward's arithmetic
// (add_layernorm_kernel).  dx = rstd (g - mean(g) - xhat mean(g xhat)) with g = dy gamma; dy xhat goes to `dyx` for dgamma.
__global__ void __launch_bounds__(256) ln_backward_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                          const float* __restrict__ gamma, const float* __restrict__ dy, int N, int C,
                                                          float eps, float* __restrict__ dx, float* __restrict__ dyx) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (n >= N) return;
    float vals[32];   // C <= 1024
    float s = 0.f;
    int cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) {
        const float x = a[(long long)n * C + c] + (b != nullptr ? b[(long long)n * C + c] : 0.f);
        vals[cnt] = x;
        s += x;
    }
    const float mean = warp_sum(s) / (float)C;
    float s2 = 0.f;
    for (int i = 0; i < cnt; ++i) { const float d = vals[i] - mean; s2 = fmaf(d, d, s2); }
    const float rstd = rsqrtf(warp_sum(s2) / (float)C + eps);
    float sg = 0.f, sgx = 0.f;
    cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) {
        const float xh = (vals[cnt] - mean) * rstd;
        const float g = dy[(long long)n * C + c];
        const float gg = g * gamma[c];
        vals[cnt] = xh;
        sg += gg;
        sgx = fmaf(gg, xh, sgx);
        dyx[(long long)n * C + c] = g * xh;
    }
    sg = warp_sum(sg) / (float)C;
    sgx = warp_sum(sgx) / (float)C;
    cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt)
        dx[(long long)n * C + c] = rstd * (dy[(long long)n * C + c] * gamma[c] - sg - vals[cnt] * sgx);
}

// ---------------------------------------------------------------------------------------------------------- L2 normalise
// y = x / max(|x|, 1e-12): dx = (dy - y (y . dy)) / |x| above the clamp, dy / 1e-12 below it (the clamp's derivative is 0)
__global__ void __launch_bounds__(256) l2n_backward_kernel(const float* __restrict__ x, const float* __restrict__ dy, int N, int C,
                                                           float* __restrict__ dx) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (n >= N) return;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = x[(long long)n * C + c]; s = fmaf(v, v, s); }
    const float raw = sqrtf(warp_sum(s));
    const float nrm = fmaxf(raw, 1e-12f);
    const bool clamped = !(raw > 1e-12f);
    float yg = 0.f;
    if (!clamped)
        for (int c = lane; c < C; c += 32) yg = fmaf(x[(long long)n * C + c] / nrm, dy[(long long)n * C + c], yg);
    yg = warp_sum(yg);
    for (int c = lane; c < C; c += 32) {
        const float g = dy[(long long)n * C + c];
        dx[(long long)n * C + c] = clamped ? g / nrm : (g - (x[(long long)n * C + c] / nrm) * yg) / nrm;
    }
}

// ---------------------------------------------------------------------------------------------------------- head_project
// dq[n][c] += dqb[n][c / d] * bp[c]   (the qb = q_h . bp_h term)
__global__ void __launch_bounds__(256) head_bias_grad_kernel(const float* __restrict__ dqb, const float* __restrict__ bp, int N, int C, int H,
                                                             float* __restrict__ dq, long long ldgq) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)N * C) return;
    const int n = (int)(t / C), c = (int)(t % C);
    float* p = dq + (long long)n * ldgq + c;
    *p = fmaf(dqb[(long long)n * H + c / (C / H)], bp[c], *p);
}

// ---------------------------------------------------------------------------------------------------------- attention
// Batched strided GEMM: C_z[i][j] = sum_t A_z(i, t) B_z(t, j), z = blockIdx.z; element (i, t) of A_z at p[z zs + i r + t c].  64 x 64
// output tile, depth 16, 4 x 4 per thread (rows ty + 16 u, columns tx + 16 v), every output summed by one thread in t order.
struct Mat {
    const float* p;
    long long r, c, zs;
};
constexpr int SG_T = 64;

__device__ __forceinline__ void sg_stage(const Mat& m, long long z, int i0, int t0, int I, int K, float (*S)[SG_T]) {
    // S[t][i] for t < 16, i < 64; the fast-moving thread index runs along whichever of i / t has unit stride
    const float* base = m.p + z * m.zs;
    const bool t_fast = (m.c == 1);
    for (int e = threadIdx.x; e < 16 * SG_T; e += 256) {
        const int tt = t_fast ? (e & 15) : (e / SG_T);
        const int ii = t_fast ? (e >> 4) : (e % SG_T);
        const int i = i0 + ii, t = t0 + tt;
        S[tt][ii] = (i < I && t < K) ? base[(long long)i * m.r + (long long)t * m.c] : 0.f;
    }
}

__global__ void __launch_bounds__(256) att_gemm_kernel(Mat A, Mat Bt, float* __restrict__ Cm, long long c_r, long long c_zs, int M, int N,
                                                       int K) {
    // Bt: element (j, t) of B^T, so both operands are staged the same way
    __shared__ float As[16][SG_T];
    __shared__ float Bs[16][SG_T];
    const long long z = blockIdx.z;
    const int i0 = blockIdx.y * SG_T, j0 = blockIdx.x * SG_T;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = 0.f;
    for (int t0 = 0; t0 < K; t0 += 16) {
        sg_stage(A, z, i0, t0, M, K, As);
        sg_stage(Bt, z, j0, t0, N, K, Bs);
        __syncthreads();
#pragma unroll
        for (int t = 0; t < 16; ++t) {
            float a[4], b[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { a[u] = As[t][ty + 16 * u]; b[u] = Bs[t][tx + 16 * u]; }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
        }
        __syncthreads();
    }
    float* out = Cm + z * c_zs;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int i = i0 + ty + 16 * u;
        if (i >= M) continue;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int j = j0 + tx + 16 * v;
            if (j < N) out[(long long)i * c_r + j] = acc[u][v];
        }
    }
}

static void att_gemm(const Mat& A, const Mat& Bt, float* Cm, long long c_r, long long c_zs, int M, int N, int K, int batch, cudaStream_t st) {
    const dim3 grid((unsigned)((N + SG_T - 1) / SG_T), (unsigned)((M + SG_T - 1) / SG_T), (unsigned)batch);
    att_gemm_kernel<<<grid, 256, 0, st>>>(A, Bt, Cm, c_r, c_zs, M, N, K);
    count_launches(1);
}

// dS'[n][h][m] = P (dP - sum_c dO O) / div in place over dP (N, H, M); one warp per (n, h).  With the structure term also
// dqb[n][h] = sum_m dS'[n][h][m].
__global__ void __launch_bounds__(256) att_softmax_grad_kernel(const float* __restrict__ P, const float* __restrict__ dO,
                                                               const float* __restrict__ O, long long ldo, int N, int M, int C, int H,
                                                               float div, float* __restrict__ dS, float* __restrict__ dqb) {
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= (long long)N * H) return;
    const int n = (int)(row / H), h = (int)(row % H), d = C / H;
    float delta = 0.f;
    for (int c = lane; c < d; c += 32) delta = fmaf(dO[(long long)n * C + h * d + c], O[(long long)n * ldo + h * d + c], delta);
    delta = warp_sum(delta);
    const float* p = P + row * M;
    float* s = dS + row * M;
    float sum = 0.f;
    for (int m = lane; m < M; m += 32) {
        const float g = p[m] * (s[m] - delta) / div;
        s[m] = g;
        sum += g;
    }
    if (dqb != nullptr) {
        sum = warp_sum(sum);
        if (lane == 0) dqb[row] = sum;
    }
}

// The E pass of one query row n per CTA: dE[n][m][:] = sum_h dS'[n][h][m] qp[n][h][:] and dqp[n][h][:] = sum_m dS'[n][h][m] E[n][m][:].
// Lanes <-> channels (lane owns channels 128 j + 4 lane .. +3), warp w takes keys w, w + 8, ... two at a time; E is read once and dE
// written once with streaming accesses; the eight warps' dqp partials are folded in warp order through shared memory.
constexpr int AEG_WARPS = 8;

template <int H, int J>
__global__ void __launch_bounds__(256) att_embed_grad_kernel(const float* __restrict__ dS, const float* __restrict__ qp,
                                                             const float* __restrict__ E, int M, float* __restrict__ dqp,
                                                             float* __restrict__ dE) {
    constexpr int C = 128 * J;
    extern __shared__ float4 aeg_smem[];
    float4* red = aeg_smem;                                                    // [warps][H][C / 4]
    float* ds_s = reinterpret_cast<float*>(aeg_smem + AEG_WARPS * H * (C / 4));   // [H][M]
    const int n = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = threadIdx.x; t < H * M; t += blockDim.x) ds_s[t] = dS[(long long)n * H * M + t];
    float4 qpv[H][J], acc[H][J];
#pragma unroll
    for (int h = 0; h < H; ++h)
#pragma unroll
        for (int j = 0; j < J; ++j) {
            qpv[h][j] = *reinterpret_cast<const float4*>(qp + ((long long)n * H + h) * C + j * 128 + 4 * lane);
            acc[h][j] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    __syncthreads();
    const float4* e_row = reinterpret_cast<const float4*>(E + (long long)n * M * C);
    float4* de_row = reinterpret_cast<float4*>(dE + (long long)n * M * C);
    for (int m0 = 2 * warp; m0 < M; m0 += 2 * AEG_WARPS) {
        const int nk = (m0 + 1 < M) ? 2 : 1;
        float4 e[2][J];
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
            for (int j = 0; j < J; ++j)
                e[u][j] = (u < nk) ? __ldcs(e_row + (long long)(m0 + u) * (C / 4) + j * 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            if (u >= nk) break;
            const int m = m0 + u;
#pragma unroll
            for (int j = 0; j < J; ++j) {
                float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int h = 0; h < H; ++h) {
                    const float s = ds_s[h * M + m];
                    g.x = fmaf(s, qpv[h][j].x, g.x); g.y = fmaf(s, qpv[h][j].y, g.y);
                    g.z = fmaf(s, qpv[h][j].z, g.z); g.w = fmaf(s, qpv[h][j].w, g.w);
                    acc[h][j].x = fmaf(s, e[u][j].x, acc[h][j].x); acc[h][j].y = fmaf(s, e[u][j].y, acc[h][j].y);
                    acc[h][j].z = fmaf(s, e[u][j].z, acc[h][j].z); acc[h][j].w = fmaf(s, e[u][j].w, acc[h][j].w);
                }
                __stcs(de_row + (long long)m * (C / 4) + j * 32 + lane, g);
            }
        }
    }
#pragma unroll
    for (int h = 0; h < H; ++h)
#pragma unroll
        for (int j = 0; j < J; ++j) red[(warp * H + h) * (C / 4) + j * 32 + lane] = acc[h][j];
    __syncthreads();
    for (int t = threadIdx.x; t < H * (C / 4); t += blockDim.x) {
        float4 s = red[t];
#pragma unroll
        for (int w = 1; w < AEG_WARPS; ++w) {                   // fixed order
            const float4 x = red[w * H * (C / 4) + t];
            s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
        }
        reinterpret_cast<float4*>(dqp + (long long)n * H * C)[t] = s;
    }
}

static size_t aeg_smem_bytes(int heads, int channels, int64_t n_key) {
    return (size_t)AEG_WARPS * heads * channels * 4 + (size_t)heads * n_key * 4;
}

template <int H, int J>
static int launch_embed_grad(const float* dS, const float* qp, const float* E, int N, int M, float* dqp, float* dE, cudaStream_t st) {
    const size_t smem = aeg_smem_bytes(H, 128 * J, M);
    if (smem > 48 * 1024 && ensure_max_smem((const void*)att_embed_grad_kernel<H, J>)) return -1;
    att_embed_grad_kernel<H, J><<<(unsigned)N, 256, smem, st>>>(dS, qp, E, M, dqp, dE);
    count_launches(1);
    return 0;
}

// ---------------------------------------------------------------------------------------------------------- structure embedding
// k*[r][o]: which of the three angle terms wins the max of channel o in row r, from the same table lookups (or direct evaluations
// beyond the table) as table_embed_kernel; the first of equal values.  One warp per row.
template <int C>
__global__ void __launch_bounds__(256) gse_kstar_kernel(const float* __restrict__ a_idx, long long n_rows, const unsigned char* __restrict__ table,
                                                        int n_d, int n_a, float inv_step, const float* __restrict__ div_term,
                                                        const float* __restrict__ Wa, const float* __restrict__ ba,
                                                        unsigned char* __restrict__ kstar) {
    using LK = gtab::Lookup<C>;
    constexpr int NV = LK::NV;
    const int lane = threadIdx.x & 31;
    const float scale = reinterpret_cast<const gtab::Header*>(table)->slope_scale;
    const unsigned char* __restrict__ ta = table + gtab::HEADER_BYTES + (size_t)n_d * LK::NODE;
    const float lim_a = (float)n_a;
    for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < n_rows; r += (long long)gridDim.x * 8) {
        float va[4 * NV], vb[4 * NV], vc[4 * NV];
        LK::term(a_idx[3 * r], ta, lim_a, inv_step, scale, div_term, Wa, ba, lane, va);
        LK::term(a_idx[3 * r + 1], ta, lim_a, inv_step, scale, div_term, Wa, ba, lane, vb);
        LK::term(a_idx[3 * r + 2], ta, lim_a, inv_step, scale, div_term, Wa, ba, lane, vc);
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            unsigned char k[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float x = va[4 * j + e], y = vb[4 * j + e], z = vc[4 * j + e];
                k[e] = (x >= y && x >= z) ? 0 : (y >= z ? 1 : 2);
            }
            *reinterpret_cast<uchar4*>(kstar + r * C + 128 * j + 4 * lane) = make_uchar4(k[0], k[1], k[2], k[3]);
        }
    }
}

// dWd[o][i] = sum_r dE[r][o] s_i(d_r), dWa[o][i] = sum_r dE[r][o] s_i(a_{r, k*(r, o)}) over one 2048-row chunk (blockIdx.z) for a
// 64 x 64 tile (o: blockIdx.y, i: blockIdx.x).  The sinusoid s(x) = [sin x w_0, cos x w_0, sin x w_1, ...] is evaluated with
// sincosf as the forward's direct path does (exact() in gse_table.cuh) and never stored.  Thread (tx, ty) owns o = o0 + 4 ty .. +3,
// i = i0 + 4 tx .. +3 of both sums.
constexpr int GB_ROWS = 2048;
constexpr int GB_T = 64;
constexpr int GB_R = 16;

template <int C>
__global__ void __launch_bounds__(256) gse_dw_partial_kernel(const float* __restrict__ dE, const float* __restrict__ d_idx,
                                                             const float* __restrict__ a_idx, const unsigned char* __restrict__ kstar,
                                                             const float* __restrict__ div_term, long long n_rows,
                                                             float* __restrict__ part) {
    __shared__ __align__(16) float Gs[GB_R][GB_T];
    __shared__ __align__(16) unsigned char Ks[GB_R][GB_T];
    __shared__ __align__(16) float Ss[GB_R][4][GB_T];                  // [row][0: d, 1..3: a_k][i]
    const int i0 = blockIdx.x * GB_T, o0 = blockIdx.y * GB_T;
    const long long r0 = (long long)blockIdx.z * GB_ROWS;
    const long long r1 = min(n_rows, r0 + GB_ROWS);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float accd[4][4], acca[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) { accd[u][v] = 0.f; acca[u][v] = 0.f; }
    for (long long rb = r0; rb < r1; rb += GB_R) {
        for (int e = threadIdx.x; e < GB_R * GB_T; e += 256) {
            const int rr = e / GB_T, c = e % GB_T;
            const long long r = rb + rr;
            const bool ok = r < r1;
            Gs[rr][c] = ok ? dE[r * C + o0 + c] : 0.f;
            Ks[rr][c] = ok ? kstar[r * C + o0 + c] : 0;
        }
        for (int e = threadIdx.x; e < GB_R * 4 * (GB_T / 2); e += 256) {
            const int rr = e / (4 * (GB_T / 2)), rem = e % (4 * (GB_T / 2));
            const int arg = rem / (GB_T / 2), f = rem % (GB_T / 2);
            const long long r = rb + rr;
            float x = 0.f;
            if (r < r1) x = arg == 0 ? d_idx[r] : a_idx[3 * r + arg - 1];
            float s, c;
            sincosf(__fmul_rn(x, div_term[i0 / 2 + f]), &s, &c);
            Ss[rr][arg][2 * f] = s;
            Ss[rr][arg][2 * f + 1] = c;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < GB_R; ++rr) {
            const float4 g = *reinterpret_cast<const float4*>(&Gs[rr][4 * ty]);
            const uchar4 k = *reinterpret_cast<const uchar4*>(&Ks[rr][4 * ty]);
            const float4 sd = *reinterpret_cast<const float4*>(&Ss[rr][0][4 * tx]);
            const float ga[4] = {g.x, g.y, g.z, g.w};
            const unsigned char ka[4] = {k.x, k.y, k.z, k.w};
            const float sda[4] = {sd.x, sd.y, sd.z, sd.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float4 sa = *reinterpret_cast<const float4*>(&Ss[rr][1 + ka[u]][4 * tx]);
                const float saa[4] = {sa.x, sa.y, sa.z, sa.w};
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    accd[u][v] = fmaf(ga[u], sda[v], accd[u][v]);
                    acca[u][v] = fmaf(ga[u], saa[v], acca[u][v]);
                }
            }
        }
        __syncthreads();
    }
    float* pd = part + (size_t)blockIdx.z * 2 * C * C;
    float* pa = pd + (size_t)C * C;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int o = o0 + 4 * ty + u;
        *reinterpret_cast<float4*>(pd + (size_t)o * C + i0 + 4 * tx) = make_float4(accd[u][0], accd[u][1], accd[u][2], accd[u][3]);
        *reinterpret_cast<float4*>(pa + (size_t)o * C + i0 + 4 * tx) = make_float4(acca[u][0], acca[u][1], acca[u][2], acca[u][3]);
    }
}

__global__ void __launch_bounds__(256) gse_dw_fold_kernel(const float* __restrict__ part, int chunks, int CC, float* __restrict__ dwd,
                                                          float* __restrict__ dwa) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * CC) return;
    double s = 0.0;
    for (int z = 0; z < chunks; ++z) s += (double)part[(size_t)z * 2 * CC + t];
    if (t < CC) dwd[t] = (float)s;
    else dwa[t - CC] = (float)s;
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_add_layernorm_backward_workspace_bytes(int64_t n, int64_t channels) {
    return align_up((size_t)n * channels * 4, 256) + atb_bytes(n, 1, channels) + 1024;
}

int geob200_add_layernorm_backward(const float* a, const float* b, const float* gamma, int64_t n, int64_t channels, float eps,
                                   const float* grad_y, float* grad_x, float* grad_gamma, float* grad_beta, void* workspace,
                                   size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n > 0 && channels > 0 && channels <= 1024, "add_layernorm_backward: bad shape (n %lld, channels %lld <= 1024)",
                 (long long)n, (long long)channels);
    GEOB_REQUIRE(a != nullptr && gamma != nullptr && grad_y != nullptr && grad_x != nullptr, "add_layernorm_backward: null input");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_add_layernorm_backward_workspace_bytes(n, channels),
                 "add_layernorm_backward: workspace too small");
    Arena ar(workspace, workspace_bytes);
    float* dyx = ar.take<float>((size_t)n * channels);
    float* part = ar.take<float>(atb_bytes(n, 1, channels) / 4 + 1);
    GEOB_REQUIRE(ar.ok(), "add_layernorm_backward: workspace accounting error");
    ln_backward_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(a, b, gamma, grad_y, (int)n, (int)channels, eps, grad_x, dyx);
    count_launches(1);
    if (grad_gamma != nullptr) atb(nullptr, 0, dyx, channels, nullptr, n, 1, channels, grad_gamma, part, st);
    if (grad_beta != nullptr) atb(nullptr, 0, grad_y, channels, nullptr, n, 1, channels, grad_beta, part, st);
    GEOB_CHECK_LAUNCH();
    return 0;
}

int geob200_l2_normalize_backward(const float* x, int64_t n, int64_t channels, const float* grad_y, float* grad_x, void* stream) {
    GEOB_REQUIRE(n > 0 && channels > 0, "l2_normalize_backward: empty input");
    GEOB_REQUIRE(x != nullptr && grad_y != nullptr && grad_x != nullptr, "l2_normalize_backward: null input");
    l2n_backward_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, grad_y, (int)n, (int)channels, grad_x);
    count_launches(1);
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_head_project_backward_workspace_bytes(int64_t n, int64_t channels, int64_t heads) {
    if (heads <= 0) return 0;
    return atb_bytes(n, channels / heads, channels) + 1024;
}

int geob200_head_project_backward(const float* q, int64_t ldq, const float* wp, const float* bp, int64_t n, int64_t channels, int64_t heads,
                                  const float* grad_qp, const float* grad_qb, float* grad_q, int64_t ldgq, float* grad_wp, float* grad_bp,
                                  void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n > 0 && heads > 0 && channels > 0 && channels % heads == 0, "head_project_backward: bad shape");
    GEOB_REQUIRE(ldq >= channels && (grad_q == nullptr || ldgq >= channels), "head_project_backward: row strides below channels");
    GEOB_REQUIRE(grad_qp != nullptr && grad_qb != nullptr && (grad_q == nullptr || (wp != nullptr && bp != nullptr)) &&
                     ((grad_wp == nullptr && grad_bp == nullptr) || q != nullptr),
                 "head_project_backward: null input");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_head_project_backward_workspace_bytes(n, channels, heads),
                 "head_project_backward: workspace too small");
    const int64_t d = channels / heads;
    Arena ar(workspace, workspace_bytes);
    float* part = ar.take<float>(atb_bytes(n, d, channels) / 4 + 1);
    GEOB_REQUIRE(ar.ok(), "head_project_backward: workspace accounting error");
    if (grad_q != nullptr) {
        // dq[n, h d + t] = sum_i dqp[n, h, i] Wp[h d + t, i]: x = dqp[:, h, :], weight = Wp rows h d .. h d + d - 1, batched over heads
        const int rc = geob200_linear_batched(grad_qp, heads * channels, channels, wp, channels, d * channels, nullptr, 0, grad_q, ldgq, d, n,
                                              d, channels, heads, 0, stream);
        if (rc != 0) return rc;
        head_bias_grad_kernel<<<(unsigned)((n * channels + 255) / 256), 256, 0, st>>>(grad_qb, bp, (int)n, (int)channels, (int)heads,
                                                                                      grad_q, ldgq);
        count_launches(1);
    }
    for (int64_t h = 0; h < heads; ++h) {
        // dWp[h d + t, i] = sum_n q[n, h d + t] dqp[n, h, i];  dbp[h d + t] = sum_n q[n, h d + t] dqb[n, h]
        if (grad_wp != nullptr) atb(q + h * d, ldq, grad_qp + h * channels, heads * channels, nullptr, n, d, channels, grad_wp + h * d * channels, part, st);
        if (grad_bp != nullptr) atb(q + h * d, ldq, grad_qb + h, heads, nullptr, n, d, 1, grad_bp + h * d, part, st);
    }
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_attention_backward_batched_workspace_bytes(const geob200_att_item_t* items, int64_t n_items, int64_t heads) {
    size_t need = 0;
    for (int64_t i = 0; i < n_items; ++i) {
        const size_t b = align_up((size_t)items[i].n_query * (size_t)items[i].n_key * (size_t)heads * sizeof(float), 256);
        need = b > need ? b : need;
    }
    return need + 1024;
}

int geob200_attention_backward_batched(const geob200_att_item_t* items, const geob200_att_grad_item_t* grads, int64_t n_items, int64_t ldq,
                                       int64_t ldk, int64_t ldv, int64_t ldo, int64_t ldgq, int64_t ldgk, int64_t ldgv, int64_t channels,
                                       int64_t heads, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(items != nullptr && grads != nullptr && n_items >= 1, "attention_backward: no items");
    GEOB_REQUIRE((channels == 128 || channels == 256) && (heads == 1 || heads == 2 || heads == 4 || heads == 8),
                 "attention_backward: channels %lld (128 or 256) / heads %lld (1, 2, 4 or 8) unsupported", (long long)channels,
                 (long long)heads);
    GEOB_REQUIRE(ldq >= channels && ldk >= channels && ldv >= channels && ldo >= channels && ldgq >= channels && ldgk >= channels &&
                     ldgv >= channels,
                 "attention_backward: row strides below channels");
    for (int64_t i = 0; i < n_items; ++i) {
        const geob200_att_item_t& it = items[i];
        const geob200_att_grad_item_t& g = grads[i];
        GEOB_REQUIRE(it.n_query > 0 && it.n_key > 0, "attention_backward: empty item %lld", (long long)i);
        GEOB_REQUIRE(it.q != nullptr && it.k != nullptr && it.v != nullptr && it.out != nullptr && g.probs != nullptr && g.grad_out != nullptr,
                     "attention_backward: null input in item %lld", (long long)i);
        GEOB_REQUIRE((it.embed == nullptr) == (it.qp == nullptr) && (it.embed == nullptr) == (it.qb == nullptr),
                     "attention_backward: qp/qb/embed must come together");
        GEOB_REQUIRE(it.embed != nullptr || (g.grad_qp == nullptr && g.grad_qb == nullptr && g.grad_embed == nullptr),
                     "attention_backward: structure-term gradients of a cross-attention item");
        GEOB_REQUIRE((g.grad_qp == nullptr) == (g.grad_embed == nullptr), "attention_backward: grad_qp and grad_embed come together");
        GEOB_REQUIRE((it.embed == nullptr || ((uintptr_t)it.embed % 16) == 0) && (it.qp == nullptr || ((uintptr_t)it.qp % 16) == 0) &&
                         (g.grad_embed == nullptr || ((uintptr_t)g.grad_embed % 16) == 0) &&
                         (g.grad_qp == nullptr || ((uintptr_t)g.grad_qp % 16) == 0),
                     "attention_backward: qp, embed and their gradients must be 16-byte aligned");
        GEOB_REQUIRE(g.grad_embed == nullptr || aeg_smem_bytes((int)heads, (int)channels, it.n_key) <= 200 * 1024,
                     "attention_backward: too many keys (%lld)", (long long)it.n_key);
    }
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_attention_backward_batched_workspace_bytes(items, n_items, heads),
                 "attention_backward: workspace too small");
    float* dS = (float*)workspace;
    const int C = (int)channels, H = (int)heads, D = C / H;
    const float div = sqrtf((float)D);           // the forward's d_model_per_head ** 0.5
    for (int64_t i = 0; i < n_items; ++i) {
        const geob200_att_item_t& it = items[i];
        const geob200_att_grad_item_t& g = grads[i];
        const int N = (int)it.n_query, M = (int)it.n_key;
        const long long HM = (long long)H * M;
        // dP[n][h][m] = dO_h[n] . v_h[m]
        att_gemm(Mat{g.grad_out, C, 1, D}, Mat{it.v, ldv, 1, D}, dS, HM, M, N, M, D, H, st);
        att_softmax_grad_kernel<<<(unsigned)(((long long)N * H + 7) / 8), 256, 0, st>>>(g.probs, g.grad_out, it.out, ldo, N, M, C, H, div, dS,
                                                                                  g.grad_qb);
        count_launches(1);
        // dV_h = P_h^T dO_h,  dQ_h = dS'_h K_h,  dK_h = dS'_h^T Q_h
        if (g.grad_v != nullptr) att_gemm(Mat{g.probs, 1, HM, M}, Mat{g.grad_out, 1, C, D}, g.grad_v, ldgv, D, M, D, N, H, st);
        if (g.grad_q != nullptr) att_gemm(Mat{dS, HM, 1, M}, Mat{it.k, 1, ldk, D}, g.grad_q, ldgq, D, N, D, M, H, st);
        if (g.grad_k != nullptr) att_gemm(Mat{dS, 1, HM, M}, Mat{it.q, 1, ldq, D}, g.grad_k, ldgk, D, M, D, N, H, st);
        if (g.grad_embed != nullptr) {
            int rc = -2;
#define LAUNCH_AEG(HV) rc = (C == 256) ? launch_embed_grad<HV, 2>(dS, it.qp, it.embed, N, M, g.grad_qp, g.grad_embed, st) \
                                       : launch_embed_grad<HV, 1>(dS, it.qp, it.embed, N, M, g.grad_qp, g.grad_embed, st)
            switch (H) {
                case 1: LAUNCH_AEG(1); break;
                case 2: LAUNCH_AEG(2); break;
                case 4: LAUNCH_AEG(4); break;
                default: LAUNCH_AEG(8); break;
            }
#undef LAUNCH_AEG
            if (rc != 0) return rc;
        }
    }
    GEOB_CHECK_LAUNCH();
    return 0;
}

size_t geob200_gse_embed_backward_workspace_bytes(int64_t n_rows, int64_t channels) {
    const int64_t chunks = (n_rows + GB_ROWS - 1) / GB_ROWS;
    return align_up((size_t)n_rows * channels, 256) + align_up((size_t)chunks * 2 * channels * channels * 4, 256) +
           atb_bytes(n_rows, 1, channels) + 1024;
}

int geob200_gse_embed_backward(const float* d_indices, const float* a_indices, int64_t n_rows, int64_t angle_k, int64_t channels,
                               const void* table, size_t table_bytes, int64_t inv_step, float d_max, float a_max, const float* div_term,
                               const float* wa, const float* ba, const float* grad_embed, float* grad_wd, float* grad_bd, float* grad_wa,
                               float* grad_ba, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    // the bias column sums (atb) take one grid z-slice per 256 rows: the tighter of the two limits
    GEOB_REQUIRE(n_rows > 0 && n_rows <= 256ll * 65535, "gse_embed_backward: bad row count %lld", (long long)n_rows);
    GEOB_REQUIRE(channels == 128 || channels == 256, "gse_embed_backward: channels %lld unsupported (128 or 256)", (long long)channels);
    GEOB_REQUIRE(angle_k == 3, "gse_embed_backward: angle_k %lld unsupported (3)", (long long)angle_k);
    GEOB_REQUIRE(inv_step >= 1 && (inv_step & (inv_step - 1)) == 0, "gse_embed_backward: inv_step must be a power of two");
    GEOB_REQUIRE(d_max > 0.f && a_max > 0.f && (double)d_max * inv_step < 1.6e7 && (double)a_max * inv_step < 1.6e7,
                 "gse_embed_backward: bad table range (d_max %g, a_max %g)", (double)d_max, (double)a_max);
    GEOB_REQUIRE(table != nullptr && table_bytes > 0 && table_bytes >= geob200_gse_table_bytes(channels, inv_step, d_max, a_max),
                 "gse_embed_backward: table buffer smaller than (channels, inv_step, d_max, a_max) imply");
    GEOB_REQUIRE(d_indices != nullptr && a_indices != nullptr && div_term != nullptr && wa != nullptr && ba != nullptr && grad_embed != nullptr &&
                     grad_wd != nullptr && grad_bd != nullptr && grad_wa != nullptr && grad_ba != nullptr,
                 "gse_embed_backward: null input");
    GEOB_REQUIRE(((uintptr_t)table & 15) == 0, "gse_embed_backward: table must be 16-byte aligned");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_gse_embed_backward_workspace_bytes(n_rows, channels),
                 "gse_embed_backward: workspace too small");
    const int C = (int)channels;
    const int64_t chunks = (n_rows + GB_ROWS - 1) / GB_ROWS;
    Arena ar(workspace, workspace_bytes);
    unsigned char* kstar = ar.take<unsigned char>((size_t)n_rows * C);
    float* part = ar.take<float>((size_t)chunks * 2 * C * C);
    float* part_b = ar.take<float>(atb_bytes(n_rows, 1, C) / 4 + 1);
    GEOB_REQUIRE(ar.ok(), "gse_embed_backward: workspace accounting error");
    const int n_d = gtab::node_count(d_max, (int)inv_step), n_a = gtab::node_count(a_max, (int)inv_step);
    const unsigned char* tb = (const unsigned char*)table;
    const long long rows_ctas = (n_rows + 7) / 8;
    const unsigned kgrid = (unsigned)(rows_ctas < (long long)num_sms() * 8 ? rows_ctas : (long long)num_sms() * 8);
    const dim3 grid((unsigned)(C / GB_T), (unsigned)(C / GB_T), (unsigned)chunks);
    if (C == 256) {
        gse_kstar_kernel<256><<<kgrid, 256, 0, st>>>(a_indices, n_rows, tb, n_d, n_a, (float)inv_step, div_term, wa, ba, kstar);
        gse_dw_partial_kernel<256><<<grid, 256, 0, st>>>(grad_embed, d_indices, a_indices, kstar, div_term, n_rows, part);
    } else {
        gse_kstar_kernel<128><<<kgrid, 256, 0, st>>>(a_indices, n_rows, tb, n_d, n_a, (float)inv_step, div_term, wa, ba, kstar);
        gse_dw_partial_kernel<128><<<grid, 256, 0, st>>>(grad_embed, d_indices, a_indices, kstar, div_term, n_rows, part);
    }
    gse_dw_fold_kernel<<<(unsigned)((2 * C * C + 255) / 256), 256, 0, st>>>(part, (int)chunks, C * C, grad_wd, grad_wa);
    count_launches(3);
    // dbd = dba = the column sums of dE
    atb(nullptr, 0, grad_embed, C, nullptr, n_rows, 1, C, grad_bd, part_b, st);
    GEOB_CHECK_CUDA(cudaMemcpyAsync(grad_ba, grad_bd, (size_t)C * 4, cudaMemcpyDeviceToDevice, st));
    GEOB_CHECK_LAUNCH();
    return 0;
}

}  // extern "C"
