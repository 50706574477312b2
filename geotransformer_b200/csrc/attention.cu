// Superpoint transformer kernels: fused multi-head attention (with the geometric structure term), residual
// LayerNorm, row L2-normalisation.
//
// Reference: geotransformer/modules/transformer/rpe_transformer.py:36-103 (self attention with relative positional
// embedding), vanilla_transformer.py:50-101 (cross attention), output_layer.py:15-21 (FFN).
//
// The reference projects the (N,M,C) embedding with proj_p ((N*M, C) x (C, C) GEMM, 9.6 GFLOP per layer and cloud at
// N=271) and then contracts it with q.  Both are linear, so the projection is moved onto q exactly:
//     q_h . (Wp e + bp)_h  =  (Wp_h^T q_h) . e  +  q_h . bp_h
// The host computes qp[n,h,:] = Wp_h^T q[n,h,:] (a tiny GEMM) and this kernel streams E once per layer:
// scores, softmax and P.V never leave the SM.  HBM/L2-bound on the E read (N*M*C*4 bytes per cloud and layer).
#include "attention.cuh"
#include "common.cuh"
#include "geob200.h"

namespace geob200 {

static bool g_att_tma = true;      // self-attention through the TMA-staged kernels of attention_tma.cu (geob200_set_attention_tma)

// R = 2 query rows per CTA (key/value rows fetched once for both).  Keys are spread over LANES: lane <-> key m, so
// every dot product over channels is a private register accumulation (no shuffles); q / qp are warp-broadcast
// shared-memory reads.  Each lane handles KPT = 2 keys per pass to halve the shared-memory traffic per FMA.
// q, k, v may be column slices of wider row-major buffers (row strides ldq, ldk, ldv in floats).
// C multiple of 4 and <= 256 (one thread per channel in the P.V phase), H <= 8 heads.
constexpr int ATT_R = 2;
constexpr int ATT_KPT = 2;
constexpr int ATT_MAXH = 8;
constexpr int ATT_KQ = 8;          // key ranges of the streaming P.V kernel (64 * ATT_KQ threads)

template <int H>
__global__ void __launch_bounds__(256) attention_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                                                        const float* __restrict__ v, int ldv, const float* __restrict__ qp,
                                                        const float* __restrict__ qb, const float* __restrict__ E, int N, int M,
                                                        int C, float div, float* __restrict__ out, int ldo) {
    extern __shared__ float sm[];
    float* q_s = sm;                            // [R][C]
    float* qp_s = q_s + ATT_R * C;              // [R][H][C]
    float* sc = qp_s + ATT_R * H * C;           // [R][H][M]
    const int n0 = blockIdx.x * ATT_R;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = C / H;
    for (int t = threadIdx.x; t < ATT_R * C; t += blockDim.x) {
        const int r = t / C, n = n0 + r;
        q_s[t] = (n < N) ? q[(long long)n * ldq + (t % C)] : 0.f;
    }
    if (qp != nullptr)
        for (int t = threadIdx.x; t < ATT_R * H * C; t += blockDim.x) {
            const int r = t / (H * C), n = n0 + r;
            qp_s[t] = (n < N) ? qp[(long long)n * H * C + (t % (H * C))] : 0.f;
        }
    __syncthreads();
    const bool has_e = (E != nullptr);
    const int r1ok = (n0 + 1 < N) ? 1 : 0;
    for (int mb = warp * 32 * ATT_KPT; mb < M; mb += 8 * 32 * ATT_KPT) {
        int mk[ATT_KPT];
        bool ok[ATT_KPT];
#pragma unroll
        for (int u = 0; u < ATT_KPT; ++u) { mk[u] = mb + u * 32 + lane; ok[u] = mk[u] < M; if (!ok[u]) mk[u] = M - 1; }
        float tot[ATT_KPT][ATT_R][H];
        // q . k : every channel belongs to exactly one head
#pragma unroll
        for (int h = 0; h < H; ++h) {
            float aq[ATT_KPT][ATT_R];
#pragma unroll
            for (int u = 0; u < ATT_KPT; ++u) { aq[u][0] = 0.f; aq[u][1] = 0.f; }
            for (int c = h * d; c < (h + 1) * d; c += 4) {
                const float4 q0 = *reinterpret_cast<const float4*>(q_s + c);
                const float4 q1 = *reinterpret_cast<const float4*>(q_s + C + c);
#pragma unroll
                for (int u = 0; u < ATT_KPT; ++u) {
                    const float4 kv = *reinterpret_cast<const float4*>(k + (long long)mk[u] * ldk + c);
                    aq[u][0] = fmaf(kv.x, q0.x, fmaf(kv.y, q0.y, fmaf(kv.z, q0.z, fmaf(kv.w, q0.w, aq[u][0]))));
                    aq[u][1] = fmaf(kv.x, q1.x, fmaf(kv.y, q1.y, fmaf(kv.z, q1.z, fmaf(kv.w, q1.w, aq[u][1]))));
                }
            }
#pragma unroll
            for (int u = 0; u < ATT_KPT; ++u) { tot[u][0][h] = aq[u][0]; tot[u][1][h] = aq[u][1]; }
        }
        // (Wp_h^T q_h) . E[n, m, :] : E is read ONCE and contracted with the H projected queries
        if (has_e) {
            float ae[ATT_KPT][ATT_R][H];
#pragma unroll
            for (int u = 0; u < ATT_KPT; ++u)
#pragma unroll
                for (int r = 0; r < ATT_R; ++r)
#pragma unroll
                    for (int h = 0; h < H; ++h) ae[u][r][h] = 0.f;
            const float* e00 = E + ((long long)n0 * M + mk[0]) * C;
            const float* e01 = E + ((long long)n0 * M + mk[1]) * C;
            const float* e10 = E + ((long long)(n0 + r1ok) * M + mk[0]) * C;
            const float* e11 = E + ((long long)(n0 + r1ok) * M + mk[1]) * C;
#pragma unroll 2
            for (int c = 0; c < C; c += 4) {
                const float4 x00 = __ldg(reinterpret_cast<const float4*>(e00 + c));
                const float4 x01 = __ldg(reinterpret_cast<const float4*>(e01 + c));
                const float4 x10 = __ldg(reinterpret_cast<const float4*>(e10 + c));
                const float4 x11 = __ldg(reinterpret_cast<const float4*>(e11 + c));
#pragma unroll
                for (int h = 0; h < H; ++h) {
                    const float4 a0 = *reinterpret_cast<const float4*>(qp_s + (0 * H + h) * C + c);
                    const float4 a1 = *reinterpret_cast<const float4*>(qp_s + (1 * H + h) * C + c);
                    ae[0][0][h] = fmaf(x00.x, a0.x, fmaf(x00.y, a0.y, fmaf(x00.z, a0.z, fmaf(x00.w, a0.w, ae[0][0][h]))));
                    ae[1][0][h] = fmaf(x01.x, a0.x, fmaf(x01.y, a0.y, fmaf(x01.z, a0.z, fmaf(x01.w, a0.w, ae[1][0][h]))));
                    ae[0][1][h] = fmaf(x10.x, a1.x, fmaf(x10.y, a1.y, fmaf(x10.z, a1.z, fmaf(x10.w, a1.w, ae[0][1][h]))));
                    ae[1][1][h] = fmaf(x11.x, a1.x, fmaf(x11.y, a1.y, fmaf(x11.z, a1.z, fmaf(x11.w, a1.w, ae[1][1][h]))));
                }
            }
#pragma unroll
            for (int u = 0; u < ATT_KPT; ++u)
#pragma unroll
                for (int r = 0; r < ATT_R; ++r)
#pragma unroll
                    for (int h = 0; h < H; ++h)
                        if (n0 + r < N) tot[u][r][h] += ae[u][r][h] + qb[(long long)(n0 + r) * H + h];
        }
#pragma unroll
        for (int u = 0; u < ATT_KPT; ++u)
            if (ok[u]) {
#pragma unroll
                for (int r = 0; r < ATT_R; ++r)
#pragma unroll
                    for (int h = 0; h < H; ++h) sc[(r * H + h) * M + mk[u]] = tot[u][r][h] / div;
            }
    }
    __syncthreads();
    // softmax over m, one warp per (row, head)
    for (int rh = warp; rh < ATT_R * H; rh += 8) {
        float* s = sc + rh * M;
        float mx = -INFINITY;
        for (int m = lane; m < M; m += 32) mx = fmaxf(mx, s[m]);
        mx = warp_max(mx);
        float sum = 0.f;
        for (int m = lane; m < M; m += 32) {
            const float e = expf(s[m] - mx);
            s[m] = e;
            sum += e;
        }
        sum = warp_sum(sum);
        for (int m = lane; m < M; m += 32) s[m] = s[m] / sum;
    }
    __syncthreads();
    // out[n][c] = sum_m P[h(c)][m] v[m][c]   (4 partial sums per thread for memory-level parallelism)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int h = c / d;
        const float* p0 = sc + (0 * H + h) * M;
        const float* p1 = sc + (1 * H + h) * M;
        float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
        int m = 0;
        for (; m + 3 < M; m += 4) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float vv = v[(long long)(m + u) * ldv + c];
                a0[u] = fmaf(p0[m + u], vv, a0[u]);
                a1[u] = fmaf(p1[m + u], vv, a1[u]);
            }
        }
        for (; m < M; ++m) {
            const float vv = v[(long long)m * ldv + c];
            a0[0] = fmaf(p0[m], vv, a0[0]);
            a1[0] = fmaf(p1[m], vv, a1[0]);
        }
        if (n0 < N) out[(long long)n0 * ldo + c] = (a0[0] + a0[1]) + (a0[2] + a0[3]);
        if (n0 + 1 < N) out[(long long)(n0 + 1) * ldo + c] = (a1[0] + a1[1]) + (a1[2] + a1[3]);
    }
}

// ---- streaming path (C = 128 or 256) ---------------------------------------------------------------------------
// The self-attention layers are bound by the single pass over E (N*M*C*4 bytes, 105 MB at N = 320, C = 256).  With
// lanes <-> keys (kernel above) every lane walks its own 1 KB row: 32 rows in flight per request, and a grid of N/2
// CTAs leaves the last wave almost empty.  Here lanes <-> CHANNELS: a warp reads one E row as 1 KB of perfectly
// coalesced float4 loads, keeps its slice of q / qp in registers, and the per-head sums of 4 keys (4*H values) are
// reduced across the warp with a transposing butterfly (4*H-1 shuffles instead of 5 per value).  The grid is
// (query, key chunk): ~600 small CTAs stream E at HBM speed; raw scores go to a (N,H,M) scratch (1.6 MB) and a second
// small kernel does softmax and P.V.
constexpr int ATS_G = 4;          // keys per butterfly group

__device__ __forceinline__ float dot4(const float4 a, const float4 b, float acc) {
    return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, fmaf(a.w, b.w, acc))));
}

constexpr int ATS_DEPTH = 3;      // E row groups in flight per warp (cp.async ring in shared memory)

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Persistent CTAs (one per resident slot); a CTA owns a contiguous range of (query, 4-key group) work units, its 4 warps take
// them round-robin.  Each warp streams the E rows of its next ATS_DEPTH-1 groups into its private shared-memory ring with
// cp.async (every lane later reads back exactly the 16-byte pieces it copied, so no barrier is needed): ~8 KB of E in flight
// per warp without spending registers on it.
template <int H, int J>
__global__ void __launch_bounds__(128) att_scores_kernel(const __grid_constant__ AttBatch b, int ldq, int ldk, float div) {
    constexpr int C = 128 * J;
    constexpr int D = C / H;
    constexpr int NV = ATS_G * H;                 // values reduced together: (key u, head h) -> v[u * H + h]
    extern __shared__ float4 ring_all[];          // [4 warps][ATS_DEPTH][ATS_G][J][32 lanes]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float4* ring = ring_all + (size_t)warp * ATS_DEPTH * ATS_G * J * 32;
    const bool has_e = (b.it[0].E != nullptr);    // a batch is all self-attention (with E) or all cross-attention
    const long long groups = b.gprefix[b.n_items];
    const long long g_begin = groups * blockIdx.x / gridDim.x, g_end = groups * (blockIdx.x + 1) / gridDim.x;
    float4 qv[J];
    float4 qpv[H][J];
    int hq[J];
#pragma unroll
    for (int j = 0; j < J; ++j) hq[j] = (j * 128 + 4 * lane) / D;
    int cp = 0, ci = 0;                           // item cursors of the prefetcher and of the consumer (work units only move forward)

    auto prefetch = [&](long long g, int slot) {           // E rows of group g -> ring slot (no-op group when g is out of range)
        if (has_e && g < g_end) {
            while (g >= b.gprefix[cp + 1]) ++cp;
            const int M = b.it[cp].M;
            const int gpq = (M + ATS_G - 1) / ATS_G;      // groups per query
            const long long gl = g - b.gprefix[cp];
            const int n = (int)(gl / gpq), m0 = (int)(gl % gpq) * ATS_G;
            const float* e_row = b.it[cp].E + (long long)n * M * C;
#pragma unroll
            for (int u = 0; u < ATS_G; ++u) {
                const int m = min(m0 + u, M - 1);
#pragma unroll
                for (int j = 0; j < J; ++j)
                    cp_async16(&ring[((slot * ATS_G + u) * J + j) * 32 + lane], e_row + (long long)m * C + j * 128 + 4 * lane);
            }
        }
        cp_async_commit();
    };

    const long long first = g_begin + warp;
#pragma unroll
    for (int d = 0; d < ATS_DEPTH - 1; ++d) prefetch(first + 4ll * d, d);
    long long n_loaded = -1;
    int slot = 0;
    for (long long g = first; g < g_end; g += 4) {
        prefetch(g + 4ll * (ATS_DEPTH - 1), (slot + ATS_DEPTH - 1) % ATS_DEPTH);
        while (g >= b.gprefix[ci + 1]) ++ci;
        const int M = b.it[ci].M;
        const int gpq = (M + ATS_G - 1) / ATS_G;
        const long long gl = g - b.gprefix[ci];
        const int n = (int)(gl / gpq), m0 = (int)(gl % gpq) * ATS_G;
        const float* __restrict__ k = b.it[ci].k;
        if ((((long long)ci << 32) | n) != n_loaded) {        // warp-uniform
            const float* __restrict__ q = b.it[ci].q;
            const float* __restrict__ qp = b.it[ci].qp;
#pragma unroll
            for (int j = 0; j < J; ++j) {
                const int c = j * 128 + 4 * lane;
                qv[j] = *reinterpret_cast<const float4*>(q + (long long)n * ldq + c);
#pragma unroll
                for (int h = 0; h < H; ++h)
                    qpv[h][j] = has_e ? *reinterpret_cast<const float4*>(qp + ((long long)n * H + h) * C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            n_loaded = ((long long)ci << 32) | n;
        }
        float4 kk[ATS_G][J];
#pragma unroll
        for (int u = 0; u < ATS_G; ++u) {
            const int m = min(m0 + u, M - 1);
#pragma unroll
            for (int j = 0; j < J; ++j) kk[u][j] = __ldg(reinterpret_cast<const float4*>(k + (long long)m * ldk + j * 128 + 4 * lane));
        }
        cp_async_wait<ATS_DEPTH - 1>();                       // this group's E rows have landed (own copies only: no barrier)
        float v[NV];
#pragma unroll
        for (int u = 0; u < ATS_G; ++u) {
#pragma unroll
            for (int h = 0; h < H; ++h) {
                float a = 0.f;
#pragma unroll
                for (int j = 0; j < J; ++j) {
                    const float p = dot4(kk[u][j], qv[j], 0.f);
                    a += (hq[j] == h) ? p : 0.f;
                    if (has_e) a = dot4(ring[((slot * ATS_G + u) * J + j) * 32 + lane], qpv[h][j], a);
                }
                v[u * H + h] = a;
            }
        }
        warp_butterfly(v, lane);      // transposing reduction: lane l ends up with value index l >> (5 - log2 NV)
        // NV = 2^b values: value index = the top b lane bits; one lane per value writes
        constexpr int SH = (NV == 32) ? 0 : (NV == 16) ? 1 : (NV == 8) ? 2 : 3;
        const int idx = lane >> SH;
        const int u = idx / H, h = idx % H;
        if ((lane & ((1 << SH) - 1)) == 0 && m0 + u < M) {
            const float bias = has_e ? b.it[ci].qb[(long long)n * H + h] : 0.f;
            b.it[ci].S[((long long)n * H + h) * M + m0 + u] = (v[0] + bias) / div;
        }
        slot = (slot + 1) % ATS_DEPTH;
    }
    cp_async_wait<0>();
}

// softmax over the keys and P.V for R = 2 queries per CTA (value rows fetched once for both); thread <-> channel
template <int H>
__global__ void __launch_bounds__(512) att_softmax_pv_kernel(const __grid_constant__ AttBatch b, int ldv, int C, int ldo) {
    extern __shared__ float sm[];
    float* sc = sm;                               // [R][H][M]
    const AttItem& item = b.it[blockIdx.y];
    const int N = item.N, M = item.M;
    const int n0 = blockIdx.x * ATT_R;
    if (n0 >= N) return;                          // grid.x covers the largest item of the batch
    const float* S = item.S;                      // overwritten by P below
    const float* __restrict__ v = item.v;
    float* __restrict__ out = item.out;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = C / H;
    for (int rh = warp; rh < ATT_R * H; rh += (int)(blockDim.x >> 5)) {
        const int r = rh / H;
        float* s = sc + rh * M;
        if (n0 + r >= N) {
            for (int m = lane; m < M; m += 32) s[m] = 0.f;
            continue;
        }
        const float* src = S + ((long long)(n0 + r) * H + (rh % H)) * M;
        float mx = -INFINITY;
        for (int m = lane; m < M; m += 32) { const float x = src[m]; s[m] = x; mx = fmaxf(mx, x); }
        mx = warp_max(mx);
        float sum = 0.f;
        for (int m = lane; m < M; m += 32) {
            const float e = expf(s[m] - mx);
            s[m] = e;
            sum += e;
        }
        sum = warp_sum(sum);
        float* dst = item.S + ((long long)(n0 + r) * H + (rh % H)) * M;      // S keeps P, as the TMA kernels leave it (backward)
        for (int m = lane; m < M; m += 32) {
            s[m] = s[m] / sum;
            dst[m] = s[m];
        }
    }
    __syncthreads();
    // P.V: thread = (4 channels, one of ATT_KQ key ranges); 16-byte value loads, 4 of them in flight; ranges folded through smem
    float4* red = reinterpret_cast<float4*>(sc + ((ATT_R * H * M + 3) & ~3));      // [4][R][C/4]
    const int C4 = C >> 2;
    const int kq = threadIdx.x / 64, c4 = threadIdx.x % 64;
    if (c4 < C4) {
        const int h = (4 * c4) / d;
        const float* p0 = sc + (0 * H + h) * M;
        const float* p1 = sc + (1 * H + h) * M;
        const int per = (M + ATT_KQ - 1) / ATT_KQ, mb = kq * per, me = min(M, mb + per);
        float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;
        int m = mb;
        for (; m + 3 < me; m += 4) {
            float4 vv[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) vv[u] = __ldg(reinterpret_cast<const float4*>(v + (long long)(m + u) * ldv) + c4);
#pragma unroll
            for (int u = 0; u < 4; u += 2) {
                const float w0 = p0[m + u], w1 = p1[m + u], x0 = p0[m + u + 1], x1 = p1[m + u + 1];
                a0.x = fmaf(w0, vv[u].x, a0.x); a0.y = fmaf(w0, vv[u].y, a0.y); a0.z = fmaf(w0, vv[u].z, a0.z); a0.w = fmaf(w0, vv[u].w, a0.w);
                a1.x = fmaf(w1, vv[u].x, a1.x); a1.y = fmaf(w1, vv[u].y, a1.y); a1.z = fmaf(w1, vv[u].z, a1.z); a1.w = fmaf(w1, vv[u].w, a1.w);
                b0.x = fmaf(x0, vv[u + 1].x, b0.x); b0.y = fmaf(x0, vv[u + 1].y, b0.y); b0.z = fmaf(x0, vv[u + 1].z, b0.z); b0.w = fmaf(x0, vv[u + 1].w, b0.w);
                b1.x = fmaf(x1, vv[u + 1].x, b1.x); b1.y = fmaf(x1, vv[u + 1].y, b1.y); b1.z = fmaf(x1, vv[u + 1].z, b1.z); b1.w = fmaf(x1, vv[u + 1].w, b1.w);
            }
        }
        for (; m < me; ++m) {
            const float4 vv = __ldg(reinterpret_cast<const float4*>(v + (long long)m * ldv) + c4);
            const float w0 = p0[m], w1 = p1[m];
            a0.x = fmaf(w0, vv.x, a0.x); a0.y = fmaf(w0, vv.y, a0.y); a0.z = fmaf(w0, vv.z, a0.z); a0.w = fmaf(w0, vv.w, a0.w);
            a1.x = fmaf(w1, vv.x, a1.x); a1.y = fmaf(w1, vv.y, a1.y); a1.z = fmaf(w1, vv.z, a1.z); a1.w = fmaf(w1, vv.w, a1.w);
        }
        red[(kq * ATT_R + 0) * C4 + c4] = make_float4(a0.x + b0.x, a0.y + b0.y, a0.z + b0.z, a0.w + b0.w);
        red[(kq * ATT_R + 1) * C4 + c4] = make_float4(a1.x + b1.x, a1.y + b1.y, a1.z + b1.z, a1.w + b1.w);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < ATT_R * C4; t += blockDim.x) {
        const int r = t / C4, cc = t % C4;
        if (n0 + r >= N) continue;
        float4 acc = red[(0 * ATT_R + r) * C4 + cc];
#pragma unroll
        for (int g = 1; g < ATT_KQ; ++g) {                      // fixed order
            const float4 x = red[(g * ATT_R + r) * C4 + cc];
            acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
        }
        float* o = out + (long long)(n0 + r) * ldo + 4 * cc;
        o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
    }
}

template <int H, int J>
static int launch_streaming(const AttBatch& b, int ldq, int ldk, int ldv, float div, int ldo, cudaStream_t st) {
    // one CTA per resident slot (occupancy queried once per instantiation); each owns a contiguous range of 4-key groups
    constexpr int ring_bytes = 4 * ATS_DEPTH * ATS_G * J * 32 * (int)sizeof(float4);
    if (ring_bytes > 48 * 1024 && ensure_max_smem((const void*)att_scores_kernel<H, J>)) return -1;
    static int per_sm = 0;          // same value on every device of the box; a racing first call computes it twice
    if (per_sm == 0) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, att_scores_kernel<H, J>, 128, ring_bytes) != cudaSuccess || per_sm < 1)
            per_sm = 1;
    }
    const long long groups = b.gprefix[b.n_items];
    long long grid = (long long)per_sm * num_sms();
    if (grid * 4 > groups) grid = (groups + 3) / 4;
    att_scores_kernel<H, J><<<(unsigned)grid, 128, ring_bytes, st>>>(b, ldq, ldk, div);
    int max_n = 0, max_m = 0;
    for (int i = 0; i < b.n_items; ++i) { max_n = b.it[i].N > max_n ? b.it[i].N : max_n; max_m = b.it[i].M > max_m ? b.it[i].M : max_m; }
    const size_t smem = sizeof(float) * (ATT_R * H * (size_t)((max_m + 3) / 4 * 4) + ATT_KQ * ATT_R * 128 * J);     // scores + the partial outputs
    if (smem > 48 * 1024 && ensure_max_smem((const void*)att_softmax_pv_kernel<H>)) return -1;
    const dim3 pv_grid((unsigned)((max_n + ATT_R - 1) / ATT_R), (unsigned)b.n_items);
    att_softmax_pv_kernel<H><<<pv_grid, 64 * ATT_KQ, smem, st>>>(b, ldv, 128 * J, ldo);
    return 0;
}

// qb[n][h] = sum_c q[n][h*d + c] * bp[h*d + c]
__global__ void __launch_bounds__(256) head_bias_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ bp, int N, int C,
                                                        int H, float* __restrict__ qb) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N * H) return;
    const int n = t / H, h = t % H, d = C / H;
    float s = 0.f;
    for (int c = 0; c < d; ++c) s = fmaf(q[(long long)n * ldq + h * d + c], bp[h * d + c], s);
    qb[t] = s;
}

// y = LayerNorm(a + b) * gamma + beta, one warp per row (torch.nn.LayerNorm, eps inside the sqrt, biased variance)
__global__ void __launch_bounds__(256) add_layernorm_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            int N, int C, float eps, float* __restrict__ y) {
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
    cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) y[(long long)n * C + c] = (vals[cnt] - mean) * rstd * gamma[c] + beta[c];
}

// F.normalize(x, p=2, dim=1): x / max(||x||, 1e-12)
__global__ void __launch_bounds__(256) l2_normalize_kernel(const float* __restrict__ x, int N, int C, float* __restrict__ y) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (n >= N) return;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = x[(long long)n * C + c]; s = fmaf(v, v, s); }
    const float nrm = fmaxf(sqrtf(warp_sum(s)), 1e-12f);
    for (int c = lane; c < C; c += 32) y[(long long)n * C + c] = x[(long long)n * C + c] / nrm;
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_attention_workspace_bytes(int64_t n_query, int64_t n_key, int64_t heads) {
    return (size_t)n_query * (size_t)n_key * (size_t)heads * sizeof(float) + 256;
}

// whether the streaming path takes an item: C = 128 / 256 and the softmax / P.V kernel's scores of one query tile fit its shared memory
static bool streaming_fits(int64_t n_key, int64_t channels, int64_t heads) {
    const size_t smem_pv = sizeof(float) * (ATT_R * heads * (size_t)((n_key + 3) / 4 * 4) + ATT_KQ * ATT_R * channels);
    return (channels == 128 || channels == 256) && smem_pv <= 200 * 1024;
}

// Streaming path for a batch of items sharing channels / heads / row strides.  Returns 1 when the shape is not handled by it.
static int attention_streaming_batch(const geob200_att_item_t* items, int64_t n_items, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                                     int64_t channels, int64_t heads, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (!(channels == 128 || channels == 256) || workspace == nullptr) return 1;
    GEOB_REQUIRE(n_items >= 1 && n_items <= ATT_MAX_ITEMS, "attention: 1..%d items per launch", ATT_MAX_ITEMS);
    AttBatch b{};
    b.n_items = (int)n_items;
    b.gprefix[0] = 0;
    b.uprefix[0] = 0;
    size_t need = 0;
    for (int i = 0; i < (int)n_items; ++i) {
        const geob200_att_item_t& it = items[i];
        GEOB_REQUIRE(it.n_query > 0 && it.n_key > 0, "attention: empty input");
        GEOB_REQUIRE((it.embed == nullptr) == (it.qp == nullptr) && (it.embed == nullptr) == (it.qb == nullptr), "attention: qp/qb/embed must come together");
        GEOB_REQUIRE((it.embed == nullptr) == (items[0].embed == nullptr), "attention: a batch is all self- or all cross-attention");
        GEOB_REQUIRE(((uintptr_t)it.q % 16) == 0 && ((uintptr_t)it.k % 16) == 0 && ((uintptr_t)it.v % 16) == 0 &&
                         (it.qp == nullptr || ((uintptr_t)it.qp % 16) == 0) && (it.embed == nullptr || ((uintptr_t)it.embed % 16) == 0),
                     "attention: q, k, v, qp, embed must be 16-byte aligned");
        if (!streaming_fits(it.n_key, channels, heads)) return 1;
        AttItem& d = b.it[i];
        d.q = it.q; d.k = it.k; d.v = it.v; d.qp = it.qp; d.qb = it.qb; d.E = it.embed; d.out = it.out;
        d.N = (int)it.n_query; d.M = (int)it.n_key;
        d.S = (float*)((char*)workspace + need);
        need += align_up((size_t)it.n_query * (size_t)it.n_key * (size_t)heads * sizeof(float), 256);
        b.gprefix[i + 1] = b.gprefix[i] + (long long)it.n_query * ((it.n_key + ATS_G - 1) / ATS_G);
        b.uprefix[i + 1] = b.uprefix[i] + (long long)it.n_query;
    }
    GEOB_REQUIRE(workspace_bytes >= need, "attention: workspace too small");
    const float div = sqrtf((float)(channels / heads));   // d_model_per_head ** 0.5
    if (g_att_tma) {
        const int rt = attention_tma_batch(b, (int)ldq, (int)ldk, (int)ldv, (int)ldo, (int)channels, (int)heads, div, st);
        if (rt <= 0) return rt;            // done, or a hard error; 1 = not handled there
    }
    int rc = -2;
#define LAUNCH_STREAM(HV)                                                                                             \
    rc = (channels == 256) ? launch_streaming<HV, 2>(b, (int)ldq, (int)ldk, (int)ldv, div, (int)ldo, st)              \
                           : launch_streaming<HV, 1>(b, (int)ldq, (int)ldk, (int)ldv, div, (int)ldo, st)
    switch (heads) {
        case 1: LAUNCH_STREAM(1); break;
        case 2: LAUNCH_STREAM(2); break;
        case 4: LAUNCH_STREAM(4); break;
        default: LAUNCH_STREAM(8); break;
    }
#undef LAUNCH_STREAM
    GEOB_REQUIRE(rc == 0, "attention: could not configure the softmax kernel");
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

static int attention_check(int64_t channels, int64_t heads, int64_t ldq, int64_t ldk, int64_t ldv) {
    GEOB_REQUIRE(channels % 4 == 0 && channels <= 256 && heads > 0 && heads <= ATT_MAXH && channels % heads == 0 &&
                     (channels / heads) % 4 == 0,
                 "attention: unsupported channels=%lld heads=%lld", (long long)channels, (long long)heads);
    GEOB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0, "attention: row strides must be multiples of 4 floats");
    GEOB_REQUIRE(heads == 1 || heads == 2 || heads == 4 || heads == 8, "attention: heads must be 1, 2, 4 or 8");
    return 0;
}

/* 1 (default): self-attention (with E) runs the TMA-staged kernels; 0: the lanes<->channels cp.async kernels */
int geob200_set_attention_tma(int on) {
    g_att_tma = on != 0;
    return 0;
}

int geob200_attention_batched_keeps_probs(const geob200_att_item_t* items, int64_t n_items, int64_t channels, int64_t heads) {
    if (items == nullptr || n_items < 1 || n_items > ATT_MAX_ITEMS) return 0;
    for (int64_t i = 0; i < n_items; ++i)
        if (items[i].n_query < 1 || items[i].n_key < 1 || !streaming_fits(items[i].n_key, channels, heads)) return 0;
    return 1;
}

size_t geob200_attention_batched_workspace_bytes(const geob200_att_item_t* items, int64_t n_items, int64_t heads) {
    size_t need = 256;
    for (int64_t i = 0; i < n_items; ++i)
        need += align_up((size_t)items[i].n_query * (size_t)items[i].n_key * (size_t)heads * sizeof(float), 256);
    return need;
}

int geob200_attention_batched(const geob200_att_item_t* items, int64_t n_items, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                              int64_t channels, int64_t heads, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (n_items == 0) return 0;
    if (attention_check(channels, heads, ldq, ldk, ldv)) return -2;
    for (int64_t i0 = 0; i0 < n_items; i0 += ATT_MAX_ITEMS) {
        const int64_t cnt = (n_items - i0 < ATT_MAX_ITEMS) ? n_items - i0 : ATT_MAX_ITEMS;
        const int rc = attention_streaming_batch(items + i0, cnt, ldq, ldk, ldv, ldo, channels, heads, workspace, workspace_bytes, st);
        if (rc < 0) return rc;
        if (rc == 1)          // shape outside the streaming path: one single-kernel launch per item
            for (int64_t i = i0; i < i0 + cnt; ++i) {
                const geob200_att_item_t& it = items[i];
                const int r2 = geob200_attention(it.q, ldq, it.k, ldk, it.v, ldv, it.qp, it.qb, it.embed, it.n_query, it.n_key, channels, heads,
                                                 it.out, ldo, nullptr, 0, stream);
                if (r2 != 0) return r2;
            }
    }
    return 0;
}

int geob200_attention(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const float* qp,
                      const float* qb, const float* embed, int64_t n_query, int64_t n_key, int64_t channels, int64_t heads,
                      float* out, int64_t ldo, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_query > 0 && n_key > 0, "attention: empty input");
    if (attention_check(channels, heads, ldq, ldk, ldv)) return -2;
    GEOB_REQUIRE((embed == nullptr) == (qp == nullptr) && (embed == nullptr) == (qb == nullptr), "attention: qp/qb/embed must come together");
    const float div = sqrtf((float)(channels / heads));   // d_model_per_head ** 0.5
    if (workspace != nullptr) {
        // streaming path: lanes <-> channels, (query, key-chunk) grid, scores through the workspace
        const geob200_att_item_t one{q, k, v, qp, qb, embed, out, n_query, n_key};
        const int rc = attention_streaming_batch(&one, 1, ldq, ldk, ldv, ldo, channels, heads, workspace, workspace_bytes, st);
        if (rc <= 0) return rc;
    }
    // generic path (any C <= 256 that is a multiple of 4; no workspace needed)
    const size_t smem = sizeof(float) * (ATT_R * channels + ATT_R * heads * channels + ATT_R * heads * n_key);
    GEOB_REQUIRE(smem <= 200 * 1024, "attention: too many keys (%lld)", (long long)n_key);
    if (smem > 48 * 1024 && (ensure_max_smem((const void*)attention_kernel<1>) || ensure_max_smem((const void*)attention_kernel<2>) ||
                             ensure_max_smem((const void*)attention_kernel<4>) || ensure_max_smem((const void*)attention_kernel<8>))) return -1;
    const unsigned grid = (unsigned)((n_query + ATT_R - 1) / ATT_R);
#define LAUNCH_ATT(HV)                                                                                                              \
    attention_kernel<HV><<<grid, 256, smem, st>>>(q, (int)ldq, k, (int)ldk, v, (int)ldv, qp, qb, embed, (int)n_query, (int)n_key,  \
                                                  (int)channels, div, out, (int)ldo)
    switch (heads) {
        case 1: LAUNCH_ATT(1); break;
        case 2: LAUNCH_ATT(2); break;
        case 4: LAUNCH_ATT(4); break;
        default: LAUNCH_ATT(8); break;
    }
#undef LAUNCH_ATT
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_head_bias(const float* q, int64_t ldq, const float* bias_p, int64_t n, int64_t channels, int64_t heads, float* qb,
                      void* stream) {
    head_bias_kernel<<<(unsigned)((n * heads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q, (int)ldq, bias_p, (int)n, (int)channels,
                                                                                          (int)heads, qb);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_add_layernorm(const float* a, const float* b, const float* gamma, const float* beta, int64_t n, int64_t channels,
                          float eps, float* y, void* stream) {
    GEOB_REQUIRE(channels <= 1024, "add_layernorm: channels > 1024");
    add_layernorm_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(a, b, gamma, beta, (int)n, (int)channels, eps, y);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_l2_normalize(const float* x, int64_t n, int64_t channels, float* y, void* stream) {
    l2_normalize_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, (int)n, (int)channels, y);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
