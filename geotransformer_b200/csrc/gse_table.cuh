// Pieces of the tabulated structure embedding (gse_table.cu) that its backward (transformer_grad.cu) recomputes with the same
// arithmetic: the table layout and the per-lane lookup / interpolation / direct evaluation of g_d and g_a.
#pragma once
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace geob200 {
namespace gtab {

constexpr int HEADER_BYTES = 256;
constexpr unsigned MAGIC = 0x47534554u;   // "GSET"

struct Header {
    unsigned magic;
    int channels;
    int inv_step;
    int n_d;
    int n_a;
    float slope_scale;       // power of two: difference = half * slope_scale
    float inv_slope_scale;
};

// Lane l of a warp owns channels 128 j + 4 l + {0..3}, j < C / 128.
template <int C>
struct Lookup {
    static constexpr int NV = C / 128;
    static constexpr int NODE = C * 6;

    // direct evaluation of W . s(x) + bias for the lane's channels (arguments beyond the table)
    static __device__ __forceinline__ void exact(float x, const float* __restrict__ div_term, const float* __restrict__ W,
                                                 const float* __restrict__ bias, int lane, float (&val)[4 * NV]) {
#pragma unroll
        for (int q = 0; q < 4 * NV; ++q) val[q] = 0.f;
        for (int f = 0; f < C / 2; ++f) {
            float s, c;
            sincosf(__fmul_rn(x, div_term[f]), &s, &c);
#pragma unroll
            for (int j = 0; j < NV; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int ch = 128 * j + 4 * lane + e;
                    const float2 w = *reinterpret_cast<const float2*>(W + (size_t)ch * C + 2 * f);
                    val[4 * j + e] = fmaf(w.y, c, fmaf(w.x, s, val[4 * j + e]));
                }
        }
#pragma unroll
        for (int j = 0; j < NV; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) val[4 * j + e] += bias[128 * j + 4 * lane + e];
    }

    // value + fraction * difference of node i, channels of this lane
    static __device__ __forceinline__ void interp(const unsigned char* __restrict__ tab, int i, float fr, int lane, float (&val)[4 * NV]) {
        const unsigned char* node = tab + (size_t)i * NODE;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const float4 f = __ldg(reinterpret_cast<const float4*>(node) + 32 * j + lane);
            const uint2 sraw = __ldg(reinterpret_cast<const uint2*>(node + C * 4) + 32 * j + lane);
            const float2 s01 = __half22float2(*reinterpret_cast<const __half2*>(&sraw.x));
            const float2 s23 = __half22float2(*reinterpret_cast<const __half2*>(&sraw.y));
            val[4 * j + 0] = fmaf(fr, s01.x, f.x);
            val[4 * j + 1] = fmaf(fr, s01.y, f.y);
            val[4 * j + 2] = fmaf(fr, s23.x, f.z);
            val[4 * j + 3] = fmaf(fr, s23.y, f.w);
        }
    }

    // one term: table when the argument is inside it, direct evaluation otherwise
    static __device__ __forceinline__ void term(float x, const unsigned char* __restrict__ tab, float lim, float inv_step, float scale,
                                                const float* __restrict__ div_term, const float* __restrict__ W,
                                                const float* __restrict__ bias, int lane, float (&val)[4 * NV]) {
        const float t = x * inv_step;
        if (t >= 0.f && t < lim) {
            const int i = (int)t;
            interp(tab, i, (t - (float)i) * scale, lane, val);
        } else {
            exact(x, div_term, W, bias, lane, val);
        }
    }

    // cold path of the embedding kernel: a row with at least one argument beyond its table
    static __device__ __noinline__ void slow_row(float4 x, const unsigned char* __restrict__ td, const unsigned char* __restrict__ ta,
                                                 float lim_d, float lim_a, float inv_step, float scale, const float* __restrict__ div_term,
                                                 const float* __restrict__ Wd, const float* __restrict__ Wa, const float* __restrict__ bd,
                                                 const float* __restrict__ ba, int lane, float* __restrict__ row) {
        float acc[4 * NV], val[4 * NV];
        term(x.y, ta, lim_a, inv_step, scale, div_term, Wa, ba, lane, acc);
        term(x.z, ta, lim_a, inv_step, scale, div_term, Wa, ba, lane, val);
#pragma unroll
        for (int q = 0; q < 4 * NV; ++q) acc[q] = fmaxf(acc[q], val[q]);
        term(x.w, ta, lim_a, inv_step, scale, div_term, Wa, ba, lane, val);
#pragma unroll
        for (int q = 0; q < 4 * NV; ++q) acc[q] = fmaxf(acc[q], val[q]);
        term(x.x, td, lim_d, inv_step, scale, div_term, Wd, bd, lane, val);
#pragma unroll
        for (int j = 0; j < NV; ++j)
            __stcs(reinterpret_cast<float4*>(row) + 32 * j + lane,
                   make_float4(val[4 * j + 0] + acc[4 * j + 0], val[4 * j + 1] + acc[4 * j + 1], val[4 * j + 2] + acc[4 * j + 2],
                               val[4 * j + 3] + acc[4 * j + 3]));
    }
};

static inline int node_count(double x_max, int inv_step) { return (int)ceil(x_max * (double)inv_step) + 1; }

}  // namespace gtab
}  // namespace geob200
