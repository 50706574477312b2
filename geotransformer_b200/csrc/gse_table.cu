// Structure embedding through tabulated projections (GeometricStructureEmbedding.forward, geotransformer.py:57-72).
//
// The reference materialises sinusoid(d_indices) (N,N,C) and sinusoid(a_indices) (N,N,k,C) and pushes them through proj_d /
// proj_a: 2 * N^2 * (1 + k) * C^2 flop per cloud (55 GF at N = 320, C = 256).  But both projections are functions of ONE scalar:
//     g_d(x) = Wd . s(x) + bd,   g_a(x) = Wa . s(x) + ba,   s(x) = [sin(x w_0), cos(x w_0), sin(x w_1), ...],  w_i <= 1,
// band-limited to 1 rad per index unit, and E[i, j, :] = g_d(d_ij) + max_k g_a(a_ijk).  So the two functions are tabulated once
// per set of weights on a uniform grid of step h = 1 / inv_step (fp64 accumulation, values stored as fp32, the forward
// difference to the next node as fp16 with one power-of-two scale for the whole table), and the embedding of a cloud becomes
// 4 lookups + 3 max + 1 add per (i, j, channel): no contraction at all, bound by the L2 reads of the nodes (6 B per channel and
// lookup) and the HBM write of E.  Linear interpolation error <= h^2 / 8 * max|g''| (< 1e-6 at h = 1/256 for unit-scale
// weights); the table is exact at the nodes to fp32 rounding.  Arguments outside the tabulated range (x >= n_nodes * h: a scene
// much larger than d_max * sigma_d) take the direct evaluation (sincosf + dot products) for that lookup, so the result never
// depends on the range chosen -- only the speed does.
//
// Table blob: [256-byte header][n_d distance nodes][n_a angle nodes]; node = C fp32 values, then C fp16 scaled differences.
#include "common.cuh"
#include "geob200.h"
#include "gse_table.cuh"

namespace geob200 {
namespace gtab {

// Bound of |g(x + h) - g(x)| <= h * sum_i w_i (|W[c][2i]| + |W[c][2i+1]|) over all channels of both projections -> the power
// of two that maps it to 2^14 (fp16 keeps 11 significant bits down to 2^-14: 28 binades below the bound).
template <int C>
__global__ void __launch_bounds__(C) table_scale_kernel(const float* __restrict__ div_term, const float* __restrict__ WdT,
                                                        const float* __restrict__ WaT, int inv_step, int n_d, int n_a,
                                                        Header* __restrict__ hdr) {
    __shared__ float red[C / 32];
    const int c = threadIdx.x;
    float bd = 0.f, ba = 0.f;
    for (int k = 0; k < C; ++k) {
        const float f = div_term[k >> 1];
        bd = fmaf(f, fabsf(WdT[(size_t)k * C + c]), bd);
        ba = fmaf(f, fabsf(WaT[(size_t)k * C + c]), ba);
    }
    float b = warp_max(fmaxf(bd, ba) / (float)inv_step);
    if ((c & 31) == 0) red[c >> 5] = b;
    __syncthreads();
    if (c == 0) {
        for (int w = 1; w < C / 32; ++w) b = fmaxf(b, red[w]);
        int e = 14;
        if (b > 0.f && b < 3.0e38f) (void)frexpf(b, &e);       // b < 2^e
        e = max(-100, min(100, e - 14));
        hdr->magic = MAGIC;
        hdr->channels = C;
        hdr->inv_step = inv_step;
        hdr->n_d = n_d;
        hdr->n_a = n_a;
        hdr->slope_scale = ldexpf(1.0f, e);
        hdr->inv_slope_scale = ldexpf(1.0f, -e);
    }
}

// One CTA per node, one thread per channel.  WT = transposed nn.Linear weight (in, out): coalesced over channels.
template <int C>
__global__ void __launch_bounds__(C) table_build_kernel(const float* __restrict__ div_term, const float* __restrict__ WdT,
                                                        const float* __restrict__ WaT, const float* __restrict__ bd,
                                                        const float* __restrict__ ba, int inv_step, int n_d,
                                                        unsigned char* __restrict__ table) {
    __shared__ double s0[C], s1[C];
    const Header* hdr = reinterpret_cast<const Header*>(table);
    const int node = blockIdx.x;
    const bool angle = node >= n_d;
    const int i = angle ? node - n_d : node;
    const float* __restrict__ WT = angle ? WaT : WdT;
    const float* __restrict__ bias = angle ? ba : bd;
    const double h = 1.0 / (double)inv_step;
    const double x0 = (double)i * h, x1 = x0 + h;
    const int t = threadIdx.x;
    if (t < C / 2) {
        const double f = (double)div_term[t];
        double s, c;
        sincos(x0 * f, &s, &c);
        s0[2 * t] = s;
        s0[2 * t + 1] = c;
        sincos(x1 * f, &s, &c);
        s1[2 * t] = s;
        s1[2 * t + 1] = c;
    }
    __syncthreads();
    double a0 = 0.0, a1 = 0.0;
    for (int k = 0; k < C; ++k) {
        const double w = (double)WT[(size_t)k * C + t];
        a0 = fma(w, s0[k], a0);
        a1 = fma(w, s1[k], a1);
    }
    unsigned char* nodep = table + HEADER_BYTES + (size_t)node * (C * 6);
    reinterpret_cast<float*>(nodep)[t] = (float)(a0 + (double)bias[t]);
    reinterpret_cast<__half*>(nodep + C * 4)[t] = __float2half_rn((float)((a1 - a0) * (double)hdr->inv_slope_scale));
}

// One warp per (anchor, point) row, 32 rows per trip: the four indices of the rows go through shared memory, every lookup is
// 1.5 KB (C = 256) of one node read by the whole warp, E is written with streaming stores (it is far larger than L2 and
// consumed by the attention layers later).
template <int C>
__global__ void __launch_bounds__(256, 4) table_embed_kernel(const float* __restrict__ d_idx, const float* __restrict__ a_idx,
                                                             long long n_pairs, const unsigned char* __restrict__ table, int n_d,
                                                             int n_a, float inv_step, const float* __restrict__ div_term,
                                                             const float* __restrict__ Wd, const float* __restrict__ Wa,
                                                             const float* __restrict__ bd, const float* __restrict__ ba,
                                                             float* __restrict__ E) {
    using LK = Lookup<C>;
    constexpr int NV = LK::NV;
    __shared__ float4 idx_s[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float scale = reinterpret_cast<const Header*>(table)->slope_scale;
    const unsigned char* __restrict__ td = table + HEADER_BYTES;
    const unsigned char* __restrict__ ta = td + (size_t)n_d * LK::NODE;
    const float lim_d = (float)n_d, lim_a = (float)n_a;
    const long long n_chunks = (n_pairs + 31) / 32;
    for (long long chunk = (long long)blockIdx.x * 8 + warp; chunk < n_chunks; chunk += (long long)gridDim.x * 8) {
        const long long p0 = chunk * 32;
        const long long p = p0 + lane;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p < n_pairs) {
            v.x = d_idx[p];
            v.y = a_idx[3 * p];
            v.z = a_idx[3 * p + 1];
            v.w = a_idx[3 * p + 2];
        }
        __syncwarp();
        idx_s[warp][lane] = v;
        __syncwarp();
        const long long left = n_pairs - p0;
        const int cnt = left < 32 ? (int)left : 32;
        for (int r = 0; r < cnt; ++r) {
            const float4 x = idx_s[warp][r];
            const float t0 = x.x * inv_step, t1 = x.y * inv_step, t2 = x.z * inv_step, t3 = x.w * inv_step;
            const bool in0 = t0 >= 0.f && t0 < lim_d, in1 = t1 >= 0.f && t1 < lim_a, in2 = t2 >= 0.f && t2 < lim_a,
                       in3 = t3 >= 0.f && t3 < lim_a;
            float* __restrict__ row = E + (p0 + r) * C;
            if (!(in0 && in1 && in2 && in3)) {       // warp-uniform: every lane sees the same four indices
                LK::slow_row(x, td, ta, lim_d, lim_a, inv_step, scale, div_term, Wd, Wa, bd, ba, lane, row);
                continue;
            }
            float vd[4 * NV], va[4 * NV], vb[4 * NV], vc[4 * NV];
            const int i0 = (int)t0, i1 = (int)t1, i2 = (int)t2, i3 = (int)t3;
            LK::interp(td, i0, (t0 - (float)i0) * scale, lane, vd);
            LK::interp(ta, i1, (t1 - (float)i1) * scale, lane, va);
            LK::interp(ta, i2, (t2 - (float)i2) * scale, lane, vb);
            LK::interp(ta, i3, (t3 - (float)i3) * scale, lane, vc);
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                float4 o;
                o.x = vd[4 * j + 0] + fmaxf(fmaxf(va[4 * j + 0], vb[4 * j + 0]), vc[4 * j + 0]);
                o.y = vd[4 * j + 1] + fmaxf(fmaxf(va[4 * j + 1], vb[4 * j + 1]), vc[4 * j + 1]);
                o.z = vd[4 * j + 2] + fmaxf(fmaxf(va[4 * j + 2], vb[4 * j + 2]), vc[4 * j + 2]);
                o.w = vd[4 * j + 3] + fmaxf(fmaxf(va[4 * j + 3], vb[4 * j + 3]), vc[4 * j + 3]);
                __stcs(reinterpret_cast<float4*>(row) + 32 * j + lane, o);
            }
        }
    }
}

}  // namespace gtab
}  // namespace geob200

using namespace geob200;

// persistent grid: 4 CTAs of 8 warps per SM, every warp walks 32-row chunks
static int table_grid(long long n_pairs) {
    const long long chunks = (n_pairs + 31) / 32;
    const long long ctas = (chunks + 7) / 8;
    const long long full = (long long)num_sms() * 4;
    return (int)(ctas < full ? ctas : full);
}

extern "C" {

size_t geob200_gse_table_bytes(int64_t channels, int64_t inv_step, float d_max, float a_max) {
    if (channels <= 0 || inv_step <= 0 || !(d_max > 0.f) || !(a_max > 0.f)) return 0;
    const size_t nodes = (size_t)gtab::node_count(d_max, (int)inv_step) + (size_t)gtab::node_count(a_max, (int)inv_step);
    return gtab::HEADER_BYTES + nodes * (size_t)channels * 6;
}

int geob200_gse_table_build(const float* div_term, const float* wd_t, const float* wa_t, const float* bd, const float* ba,
                            int64_t channels, int64_t inv_step, float d_max, float a_max, void* table, size_t table_bytes,
                            void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(channels == 128 || channels == 256, "gse_table_build: channels %lld unsupported (128 or 256)", (long long)channels);
    GEOB_REQUIRE(inv_step >= 1 && inv_step <= 65536 && (inv_step & (inv_step - 1)) == 0,
                 "gse_table_build: inv_step %lld must be a power of two", (long long)inv_step);
    GEOB_REQUIRE(d_max > 0.f && a_max > 0.f && (double)d_max * inv_step < 1.6e7 && (double)a_max * inv_step < 1.6e7,
                 "gse_table_build: bad range");
    GEOB_REQUIRE(table_bytes >= geob200_gse_table_bytes(channels, inv_step, d_max, a_max), "gse_table_build: table buffer too small");
    GEOB_REQUIRE(((uintptr_t)table & 15) == 0, "gse_table_build: table must be 16-byte aligned");
    const int n_d = gtab::node_count(d_max, (int)inv_step), n_a = gtab::node_count(a_max, (int)inv_step);
    unsigned char* tb = (unsigned char*)table;
    if (channels == 256) {
        gtab::table_scale_kernel<256><<<1, 256, 0, st>>>(div_term, wd_t, wa_t, (int)inv_step, n_d, n_a, (gtab::Header*)tb);
        gtab::table_build_kernel<256><<<(unsigned)(n_d + n_a), 256, 0, st>>>(div_term, wd_t, wa_t, bd, ba, (int)inv_step, n_d, tb);
    } else {
        gtab::table_scale_kernel<128><<<1, 128, 0, st>>>(div_term, wd_t, wa_t, (int)inv_step, n_d, n_a, (gtab::Header*)tb);
        gtab::table_build_kernel<128><<<(unsigned)(n_d + n_a), 128, 0, st>>>(div_term, wd_t, wa_t, bd, ba, (int)inv_step, n_d, tb);
    }
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

int geob200_gse_embed_table(const float* d_indices, const float* a_indices, int64_t n_rows, int64_t channels, const void* table,
                            size_t table_bytes, int64_t inv_step, float d_max, float a_max, const float* div_term, const float* wd,
                            const float* wa, const float* bd, const float* ba, float* embeddings, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(n_rows > 0, "gse_embed_table: bad shape");
    GEOB_REQUIRE(channels == 128 || channels == 256, "gse_embed_table: channels %lld unsupported (128 or 256)", (long long)channels);
    GEOB_REQUIRE(inv_step >= 1 && (inv_step & (inv_step - 1)) == 0, "gse_embed_table: inv_step must be a power of two");
    GEOB_REQUIRE(table_bytes >= geob200_gse_table_bytes(channels, inv_step, d_max, a_max) && table_bytes > 0,
                 "gse_embed_table: table buffer smaller than (channels, inv_step, d_max, a_max) imply");
    GEOB_REQUIRE(((uintptr_t)table & 15) == 0 && ((uintptr_t)embeddings & 15) == 0, "gse_embed_table: table / embeddings must be 16-byte aligned");
    const int n_d = gtab::node_count(d_max, (int)inv_step), n_a = gtab::node_count(a_max, (int)inv_step);
    const int grid = table_grid((long long)n_rows);
    const unsigned char* tb = (const unsigned char*)table;
    if (channels == 256)
        gtab::table_embed_kernel<256><<<grid, 256, 0, st>>>(d_indices, a_indices, (long long)n_rows, tb, n_d, n_a, (float)inv_step, div_term,
                                                            wd, wa, bd, ba, embeddings);
    else
        gtab::table_embed_kernel<128><<<grid, 256, 0, st>>>(d_indices, a_indices, (long long)n_rows, tb, n_d, n_a, (float)inv_step, div_term,
                                                            wd, wa, bd, ba, embeddings);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
