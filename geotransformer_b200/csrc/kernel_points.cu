// KPConv kernel-point dispositions on the device: the reference's potential descent (kernel_point_optimization_debug,
// modules/kpconv/kernel_points.py:247-386, fixed='center', 3-D) and the per-instance rotation, noise and scaling of load_kernels
// (kernel_points.py:423-455).
//
// The descent is fp64 and follows numpy's operation order step by step (sequential sums, a division per component, no FMA
// contraction: every product and sum is an explicit _rn intrinsic).  The one operation that is not bit-identical is d2^1.5:
// CUDA's pow is accurate to 2 ulp, glibc's to under 1, so a last-bit difference can occur; the descent damps such differences,
// and the stop iteration and best candidate agree with the numpy restatement on the seeds the tests cover, but that is measured,
// not guaranteed by construction.  All candidates live in one CTA: the reference's stopping test is a maximum over every
// candidate's non-centre points, i.e. a block reduction per iteration.
//
// Random draws are Philox4x32-10 with key (seed low word, seed high word):
//   initial point n:  counters (n, 0, KP_TAG_INIT, 0) -> x from words 0-1, y from words 2-3; (n, 1, KP_TAG_INIT, 0) -> z from words 0-1;
//                     u = (64-bit word >> 11) * 2^-53, coordinate 2u - 1, kept when x^2 + y^2 + z^2 < 0.5 (kernel_points.py:287-293)
//   instance layer l: theta = 2 pi u with u from counter (l, 0xFFFFFFFF, KP_TAG_INSTANCE, 0); point j's noise is Box-Muller of
//                     counters (l, j, KP_TAG_INSTANCE, 0) (x, y) and (l, j, KP_TAG_INSTANCE, 1) (z), times 0.01
#include "common.cuh"
#include "philox.cuh"
#include "geob200.h"

namespace geob200 {
namespace {

constexpr int KP_THREADS = 512;
constexpr int KP_PER_THREAD = 3;
constexpr int KP_MAX_ITEMS = KP_THREADS * KP_PER_THREAD;
constexpr int KP_MAX_ITER = 10000;
constexpr uint32_t KP_TAG_INIT = 0x4B500001u;
constexpr uint32_t KP_TAG_INSTANCE = 0x4B500002u;

__device__ __forceinline__ double u53(uint32_t lo, uint32_t hi) {
    return (double)((((uint64_t)hi << 32) | lo) >> 11) * 0x1.0p-53;
}

__device__ __forceinline__ double sum_sq3(double a, double b, double c) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c));
}

// maximum over the block; every thread gets the result (two barriers)
__device__ double block_max(double v, double* red) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double m = red[0];
    for (int w = 1; w < KP_THREADS / 32; ++w) m = fmax(m, red[w]);
    __syncthreads();
    return m;
}

__global__ void __launch_bounds__(KP_THREADS, 1)
kernel_point_optimize_kernel(const double* __restrict__ init, int K, int N, uint32_t k0, uint32_t k1, double ratio,
                             double* __restrict__ out, int* __restrict__ info) {
    __shared__ double pts[KP_MAX_ITEMS * 3];
    __shared__ double red[KP_THREADS / 32];
    __shared__ int warp_count[KP_THREADS / 32];
    const int M = K * N, t = threadIdx.x, lane = t & 31, warp = t >> 5;

    if (init != nullptr) {
        for (int i = t; i < 3 * M; i += KP_THREADS) pts[i] = init[i];
    } else {
        // draw in rounds of KP_THREADS points; accepted points keep their draw order (block-wide ordered compaction)
        int filled = 0;
        for (uint32_t round = 0; filled < M; ++round) {
            const uint32_t n = round * KP_THREADS + t;
            uint32_t a[4] = {n, 0u, KP_TAG_INIT, 0u}, b[4] = {n, 1u, KP_TAG_INIT, 0u};
            philox4x32_10(a, k0, k1);
            philox4x32_10(b, k0, k1);
            const double x = __dsub_rn(__dmul_rn(u53(a[0], a[1]), 2.0), 1.0);
            const double y = __dsub_rn(__dmul_rn(u53(a[2], a[3]), 2.0), 1.0);
            const double z = __dsub_rn(__dmul_rn(u53(b[0], b[1]), 2.0), 1.0);
            const bool ok = sum_sq3(x, y, z) < 0.5;
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) warp_count[warp] = __popc(bal);
            __syncthreads();
            int off = filled + __popc(bal & ((1u << lane) - 1u)), total = 0;
            for (int w = 0; w < KP_THREADS / 32; ++w) {
                if (w < warp) off += warp_count[w];
                total += warp_count[w];
            }
            if (ok && off < M) { pts[3 * off] = x; pts[3 * off + 1] = y; pts[3 * off + 2] = z; }
            __syncthreads();
            filled += total;
        }
    }
    __syncthreads();
    for (int i = t; i < 3 * K; i += KP_THREADS) pts[(i / 3) * N * 3 + i % 3] *= 0.0;     // kernel_points[:, 0, :] *= 0
    __syncthreads();

    double old[KP_PER_THREAD], nrm[KP_PER_THREAD], g[KP_PER_THREAD][3];
#pragma unroll
    for (int q = 0; q < KP_PER_THREAD; ++q) old[q] = 0.0;
    double moving_factor = 1e-2;
    int stop = KP_MAX_ITER;
    for (int it = 0; it < KP_MAX_ITER; ++it) {
        double dev = 0.0;
#pragma unroll
        for (int q = 0; q < KP_PER_THREAD; ++q) {
            const int m = t + q * KP_THREADS;
            if (m >= M) continue;
            const int j = m % N, base = (m - j) * 3;
            const double xj = pts[3 * m], yj = pts[3 * m + 1], zj = pts[3 * m + 2];
            double ax = 0.0, ay = 0.0, az = 0.0;
            // inter_grads[k, j] = sum over i of (x_i - x_j) / (d2^1.5 + 1e-6), i in order (numpy's axis-1 sum)
            for (int i = 0; i < N; ++i) {
                const double dx = __dsub_rn(pts[base + 3 * i], xj), dy = __dsub_rn(pts[base + 3 * i + 1], yj),
                             dz = __dsub_rn(pts[base + 3 * i + 2], zj);
                const double den = __dadd_rn(pow(sum_sq3(dx, dy, dz), 1.5), 1e-6);
                const double tx = __ddiv_rn(dx, den), ty = __ddiv_rn(dy, den), tz = __ddiv_rn(dz, den);
                if (i == 0) { ax = tx; ay = ty; az = tz; }
                else { ax = __dadd_rn(ax, tx); ay = __dadd_rn(ay, ty); az = __dadd_rn(az, tz); }
            }
            g[q][0] = __dadd_rn(ax, __dmul_rn(10.0, xj));
            g[q][1] = __dadd_rn(ay, __dmul_rn(10.0, yj));
            g[q][2] = __dadd_rn(az, __dmul_rn(10.0, zj));
            nrm[q] = __dsqrt_rn(sum_sq3(g[q][0], g[q][1], g[q][2]));
            if (j > 0) dev = fmax(dev, fabs(__dsub_rn(old[q], nrm[q])));
        }
        // every thread has read the points of this iteration once block_max returns
        if (block_max(dev, red) < 1e-5) { stop = it; break; }
#pragma unroll
        for (int q = 0; q < KP_PER_THREAD; ++q) {
            const int m = t + q * KP_THREADS;
            if (m >= M) continue;
            old[q] = nrm[q];
            const double dist = (m % N == 0) ? 0.0 : fmin(__dmul_rn(moving_factor, nrm[q]), 0.05);
            const double den = __dadd_rn(nrm[q], 1e-6);
#pragma unroll
            for (int c = 0; c < 3; ++c) pts[3 * m + c] = __dsub_rn(pts[3 * m + c], __ddiv_rn(__dmul_rn(dist, g[q][c]), den));
        }
        __syncthreads();
        moving_factor = __dmul_rn(moving_factor, 0.9995);
    }

    // rescale: ratio / (mean radius of every candidate's non-centre points)
    double rsum = 0.0;
    for (int m = t; m < M; m += KP_THREADS)
        if (m % N) rsum += __dsqrt_rn(sum_sq3(pts[3 * m], pts[3 * m + 1], pts[3 * m + 2]));
    for (int o = 16; o; o >>= 1) rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
    if (lane == 0) red[warp] = rsum;
    __syncthreads();
    double total = 0.0;
    for (int w = 0; w < KP_THREADS / 32; ++w) total += red[w];
    const double scale = ratio / (total / (double)(K * (N - 1)));
    for (int i = t; i < 3 * M; i += KP_THREADS) out[i] = pts[i] * scale;

    // load_kernels picks argmin of the last row of the saved max norms, which is zero for every candidate (so candidate 0)
    // unless the descent ran all KP_MAX_ITER iterations; then it is each candidate's max norm of the final iteration
    if (t == 0) {
        info[0] = 0;
        info[1] = stop;
    }
    if (stop == KP_MAX_ITER) {
        // each candidate's max norm of the final iteration, reduced through shared memory (the points have been written out)
        __syncthreads();
        double* last = pts;
#pragma unroll
        for (int q = 0; q < KP_PER_THREAD; ++q) {
            const int m = t + q * KP_THREADS;
            if (m < M) last[m] = old[q];
        }
        __syncthreads();
        if (t == 0) {
            int best = 0;
            double best_v = 0.0;
            for (int k = 0; k < K; ++k) {
                double v = last[k * N];
                for (int j = 1; j < N; ++j) v = fmax(v, last[k * N + j]);
                if (k == 0 || v < best_v) { best_v = v; best = k; }
            }
            info[0] = best;
        }
    }
}

__device__ __forceinline__ void box_muller(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, double& a, double& b) {
    const double u1 = 1.0 - u53(w0, w1), u2 = u53(w2, w3);      // u1 in (0, 1]
    const double r = sqrt(-2.0 * log(u1));
    double s, c;
    sincospi(2.0 * u2, &s, &c);
    a = r * c;
    b = r * s;
}

__global__ void __launch_bounds__(32)
kernel_point_instances_kernel(const double* __restrict__ disposition, int N, const double* __restrict__ radii,
                              const int64_t* __restrict__ layer_ids, uint32_t k0, uint32_t k1, float* __restrict__ out) {
    const int l = blockIdx.x, j = threadIdx.x;
    if (j >= N) return;
    const uint32_t id = (uint32_t)layer_ids[l];
    uint32_t th[4] = {id, 0xFFFFFFFFu, KP_TAG_INSTANCE, 0u};
    philox4x32_10(th, k0, k1);
    const double theta = u53(th[0], th[1]) * 2.0 * 3.141592653589793;
    const float c = (float)cos(theta), s = (float)sin(theta);
    uint32_t a[4] = {id, (uint32_t)j, KP_TAG_INSTANCE, 0u}, b[4] = {id, (uint32_t)j, KP_TAG_INSTANCE, 1u};
    philox4x32_10(a, k0, k1);
    philox4x32_10(b, k0, k1);
    double nx, ny, nz, unused;
    box_muller(a[0], a[1], a[2], a[3], nx, ny);
    box_muller(b[0], b[1], b[2], b[3], nz, unused);
    const double r = radii[l];
    // load_kernels: fp32 disposition + N(0, 0.01^2) noise, times the radius, then row vector times R (rotation about z)
    const double x = r * ((double)(float)disposition[3 * j] + 0.01 * nx);
    const double y = r * ((double)(float)disposition[3 * j + 1] + 0.01 * ny);
    const double z = r * ((double)(float)disposition[3 * j + 2] + 0.01 * nz);
    float* o = out + ((size_t)l * N + j) * 3;
    o[0] = (float)(x * c + y * s);
    o[1] = (float)(y * c - x * s);
    o[2] = (float)z;
}

}  // namespace
}  // namespace geob200

using namespace geob200;

extern "C" {

int geob200_kernel_point_optimize(const double* init, int64_t num_kernels, int64_t num_points, uint64_t seed, double ratio,
                                  double* points, int32_t* info, void* stream) {
    GEOB_REQUIRE(num_kernels >= 1 && num_points >= 2 && num_points <= GEOB200_KP_MAX_POINTS,
                 "kernel_point_optimize: num_kernels must be >= 1 and num_points in 2..%d", GEOB200_KP_MAX_POINTS);
    GEOB_REQUIRE(num_kernels * num_points <= KP_MAX_ITEMS, "kernel_point_optimize: num_kernels * num_points must be <= %d",
                 KP_MAX_ITEMS);
    GEOB_REQUIRE(ratio > 0.0, "kernel_point_optimize: ratio must be positive");
    GEOB_REQUIRE(points != nullptr && info != nullptr, "kernel_point_optimize: null output");
    kernel_point_optimize_kernel<<<1, KP_THREADS, 0, (cudaStream_t)stream>>>(init, (int)num_kernels, (int)num_points, (uint32_t)seed,
                                                                           (uint32_t)(seed >> 32), ratio, points, info);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_kernel_point_instances(const double* disposition, int64_t num_points, const double* radii, const int64_t* layer_ids,
                                   int64_t num_layers, uint64_t seed, float* out, void* stream) {
    GEOB_REQUIRE(num_points >= 1 && num_points <= GEOB200_KP_MAX_POINTS, "kernel_point_instances: num_points must be in 1..%d",
                 GEOB200_KP_MAX_POINTS);
    GEOB_REQUIRE(num_layers >= 1 && num_layers <= 65535, "kernel_point_instances: num_layers must be in 1..65535");
    GEOB_REQUIRE(disposition != nullptr && radii != nullptr && layer_ids != nullptr && out != nullptr,
                 "kernel_point_instances: null pointer");
    kernel_point_instances_kernel<<<(unsigned)num_layers, 32, 0, (cudaStream_t)stream>>>(disposition, (int)num_points, radii, layer_ids,
                                                                                       (uint32_t)seed, (uint32_t)(seed >> 32), out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
