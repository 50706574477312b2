// Training-data augmentation on the device: the per-iteration pair augmentation of the reference's 3DMatch and KITTI training
// sets and the ModelNet pair synthesis from one raw shape.
//
// Reference: geotransformer/datasets/registration/threedmatch/dataset.py (_load_point_cloud, _augment_point_cloud),
//            geotransformer/datasets/registration/kitti/dataset.py (_load_point_cloud, _augment_point_cloud),
//            geotransformer/datasets/registration/modelnet/dataset.py (__getitem__) and geotransformer/transforms/functional.py.
// Semantics and random streams: include/geob200.h and DESIGN.md section 3b.  Every draw is Philox4x32-10 keyed by
// (seed, tag of stream and cloud) with counter (index, iteration, pair_base + p), so the result is a function of the inputs and
// (seed, iteration, pair id) only -- never of the launch geometry or the rest of the batch.  The per-point arithmetic of the
// 3DMatch / KITTI modes is fp64 with explicit roundings (__dmul_rn / __dadd_rn: no contraction) and one rounding to fp32, so its
// numpy restatement (oracle/augment_oracle.py) reproduces it bit for bit.  No float atomics.
//
// ModelNet's validation and test pairs (deterministic=True) are the exception: the reference seeds numpy's global generator with
// the pair's dataset index, so modelnet_benchmark_kernel draws from numpy's own legacy stream (numpy_random.cuh) in the reference's
// order and reproduces its pairs bit for bit (oracle/modelnet_benchmark_oracle.py).
// The rotated 3DMatch / 3DLoMatch benchmark follows the same convention: the pair of dataset index i draws its two rotations from
// np.random.seed(i) (rotated_draws_kernel; oracle/rotated_oracle.py restates it in numpy).
#include "common.cuh"
#include "compaction.cuh"
#include "geob200.h"
#include "philox.cuh"
#include "numpy_random.cuh"
#include "radix_select.cuh"

namespace geob200 {

constexpr int AUG_THREADS = 1024;          // chunk_rank needs 32 warps
constexpr int AUG_POINT_THREADS = 256;
constexpr int MN_THREADS = 512;
constexpr int AUG_RECORD = 20;             // [u0 .. u10 | R row-major]
constexpr int MN_MAX_SHAPE = 8192;
constexpr int MN_MAX_POINTS = 4096;

// stream tags, XORed into the high key word; tag 0 is the target sampler's and RANSAC's key
enum AugStream : uint32_t { AUG_PAIR = 1, AUG_LIMIT = 2, AUG_NOISE = 3, AUG_SAMPLE = 4, AUG_JITTER = 5 };
__host__ __device__ constexpr uint32_t aug_tag(uint32_t stream, uint32_t cloud) { return GEOB200_AUGMENT_TAG_BASE | (stream << 4) | cloud; }

struct AugKey {
    uint32_t k0, k1, it_lo, it_hi;
};

__device__ __forceinline__ void aug_words(uint32_t w[4], uint32_t index, uint32_t pair, const AugKey& k, uint32_t tag) {
    w[0] = index; w[1] = k.it_lo; w[2] = k.it_hi; w[3] = pair;
    philox4x32_10(w, k.k0, k.k1 ^ tag);
}

// 53-bit uniform in [0, 1) from two words: ((a >> 5) 2^26 + (b >> 6)) 2^-53, exact
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
    return __dmul_rn(__dadd_rn(__dmul_rn((double)(a >> 5), 67108864.0), (double)(b >> 6)), 0x1p-53);
}
__device__ __forceinline__ double u32(uint32_t w) { return __dmul_rn((double)w, 0x1p-32); }

// the per-pair uniforms u0 .. u_{n-1} (n <= 11): Philox call i (counter index i) gives u_{2i} from words 0, 1 and u_{2i+1} from
// words 2, 3; unused slots are 0
__device__ __forceinline__ void pair_uniforms(double (&u)[11], int n, uint32_t pair, const AugKey& k) {
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        uint32_t w[4];
        aug_words(w, (uint32_t)i, pair, k, aug_tag(AUG_PAIR, 0));
        u[2 * i] = 2 * i < n ? u53(w[0], w[1]) : 0.0;
        if (2 * i + 1 < 11) u[2 * i + 1] = 2 * i + 1 < n ? u53(w[2], w[3]) : 0.0;
    }
}

// scipy Rotation.from_euler('zyx', (a, b, c)).as_matrix(), extrinsic: Rx(c) Ry(b) Rz(a), row-major
__device__ __forceinline__ void euler_zyx(double a, double b, double c, double (&R)[9]) {
    double sa, ca, sb, cb, sc, cc;
    sincos(a, &sa, &ca); sincos(b, &sb, &cb); sincos(c, &sc, &cc);
    R[0] = __dmul_rn(cb, ca);
    R[1] = -__dmul_rn(cb, sa);
    R[2] = sb;
    R[3] = __dadd_rn(__dmul_rn(cc, sa), __dmul_rn(__dmul_rn(sc, sb), ca));
    R[4] = __dsub_rn(__dmul_rn(cc, ca), __dmul_rn(__dmul_rn(sc, sb), sa));
    R[5] = -__dmul_rn(sc, cb);
    R[6] = __dsub_rn(__dmul_rn(sc, sa), __dmul_rn(__dmul_rn(cc, sb), ca));
    R[7] = __dadd_rn(__dmul_rn(sc, ca), __dmul_rn(__dmul_rn(cc, sb), sa));
    R[8] = __dmul_rn(cc, cb);
}

// row i of M times v: (M[i,0] v0 + M[i,1] v1) + M[i,2] v2
__device__ __forceinline__ double row_dot(const double* M, int i, double v0, double v1, double v2) {
    return __dadd_rn(__dadd_rn(__dmul_rn(M[3 * i], v0), __dmul_rn(M[3 * i + 1], v1)), __dmul_rn(M[3 * i + 2], v2));
}
// column i of M times v: (M[0,i] v0 + M[1,i] v1) + M[2,i] v2
__device__ __forceinline__ double col_dot(const double* M, int i, double v0, double v1, double v2) {
    return __dadd_rn(__dadd_rn(__dmul_rn(M[i], v0), __dmul_rn(M[3 + i], v1)), __dmul_rn(M[6 + i], v2));
}

__device__ __forceinline__ void write_record(double* rec, const double (&u)[11], const double (&R)[9]) {
#pragma unroll
    for (int i = 0; i < 11; ++i) rec[i] = u[i];
#pragma unroll
    for (int i = 0; i < 9; ++i) rec[11 + i] = R[i];
}

// ---- 3DMatch / KITTI ---------------------------------------------------------------------------------------------------------

// Point limit, grid (1, 2B), AUG_THREADS.  Cloud c with n <= limit: origin = 0 .. n-1.  Otherwise the `limit` smallest keys
// (philox(j) << 32) | j, written in ascending j.  word: workspace, In.start[c] + j.
__global__ void __launch_bounds__(AUG_THREADS) point_limit_kernel(const __grid_constant__ Segs In, const __grid_constant__ Segs Out,
                                                                 int B, int limit, AugKey key, uint32_t pair_base,
                                                                 uint32_t* __restrict__ word, int* __restrict__ origin) {
    __shared__ unsigned hist[256];
    __shared__ unsigned prefix_s, kth_s;
    __shared__ int warp_tot[32];
    const int c = blockIdx.y, n = In.count[c];
    const uint32_t pair = pair_base + (uint32_t)(c % B), tag = aug_tag(AUG_LIMIT, c >= B ? 1u : 0u);
    int* out = origin + Out.start[c];
    if (n <= limit) {
        for (int j = threadIdx.x; j < n; j += AUG_THREADS) out[j] = j;
        return;
    }
    word += In.start[c];
    for (int j = threadIdx.x; j < n; j += AUG_THREADS) {
        uint32_t w[4];
        aug_words(w, (uint32_t)j, pair, key, tag);
        word[j] = w[0];
    }
    __syncthreads();
    // the `limit` smallest (word, j) = the `limit` largest ~word, ties at the threshold to the lowest j
    unsigned thr;
    int need_eq;
    radix_select_kth((long long)n, limit, [&](long long j) { return ~word[j]; }, hist, &prefix_s, &kth_s, thr, need_eq);
    int kept = 0, eq = 0;
    for (int base = 0; base < n; base += AUG_THREADS) {
        const int j = base + threadIdx.x;
        const unsigned b = j < n ? ~word[j] : 0u;
        const bool fe = j < n && b == thr;
        int te;
        const int re = chunk_rank(fe, warp_tot, &te);
        const bool f = j < n && (b > thr || (fe && eq + re < need_eq));
        int tot;
        const int r = chunk_rank(f, warp_tot, &tot);
        if (f) out[kept + r] = j;
        kept += tot; eq += te;
    }
}

struct AugParams {
    int mode;
    double noise, rotation_factor, min_scale, max_scale, shift;
};

// Per-point pass, grid (ceil(Out.max / AUG_POINT_THREADS), 2B).  Thread 0 of every CTA draws its pair's uniforms and R (a few
// Philox calls); the first CTA of each ref cloud also writes the pair's record and transform.
__global__ void __launch_bounds__(AUG_POINT_THREADS) augment_points_kernel(
        const float* __restrict__ points, const __grid_constant__ Segs In, const __grid_constant__ Segs Out,
        const int* __restrict__ origin, const float* __restrict__ T_in, int B, AugParams P, AugKey key, uint32_t pair_base,
        float* __restrict__ out, float* __restrict__ T_out, double* __restrict__ record) {
    __shared__ double prm[16];             // R (9), this cloud rotated, scale, shift (3)
    const int c = blockIdx.y, p = c % B;
    const bool src = c >= B, kitti = P.mode == GEOB200_AUGMENT_KITTI;
    const uint32_t pair = pair_base + (uint32_t)p;
    if (threadIdx.x == 0) {
        double u[11], R[9];
        pair_uniforms(u, kitti ? 11 : 4, pair, key);
        // numpy: rand(3) * pi * 2 / rotation_factor
        euler_zyx(__ddiv_rn(__dmul_rn(__dmul_rn(u[0], M_PI), 2.0), P.rotation_factor),
                  __ddiv_rn(__dmul_rn(__dmul_rn(u[1], M_PI), 2.0), P.rotation_factor),
                  __ddiv_rn(__dmul_rn(__dmul_rn(u[2], M_PI), 2.0), P.rotation_factor), R);
        const bool rot_ref = u[3] > 0.5;
        // numpy: min + (max - min) * u;  uniform(-s, s) = -s + (s - -s) * u
        const double scale = kitti ? __dadd_rn(P.min_scale, __dmul_rn(__dsub_rn(P.max_scale, P.min_scale), u[4])) : 1.0;
        const double w2 = __dsub_rn(P.shift, -P.shift);
        double rs[3], ss[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            rs[i] = kitti ? __dadd_rn(-P.shift, __dmul_rn(w2, u[5 + i])) : 0.0;
            ss[i] = kitti ? __dadd_rn(-P.shift, __dmul_rn(w2, u[8 + i])) : 0.0;
        }
#pragma unroll
        for (int i = 0; i < 9; ++i) prm[i] = R[i];
        prm[9] = (src ? !rot_ref : rot_ref) ? 1.0 : 0.0;
        prm[10] = scale;
#pragma unroll
        for (int i = 0; i < 3; ++i) prm[11 + i] = src ? ss[i] : rs[i];
        if (!src && blockIdx.x == 0) {
            write_record(record + (long long)p * AUG_RECORD, u, R);
            double G[9], g[3], N[9], t[3];
            const float* T = T_in + 16ll * p;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
#pragma unroll
                for (int j = 0; j < 3; ++j) G[3 * i + j] = (double)T[4 * i + j];
                g[i] = (double)T[4 * i + 3];
            }
            if (rot_ref) {                 // rotation = R_aug R_gt, translation = R_aug t_gt
#pragma unroll
                for (int i = 0; i < 3; ++i) {
#pragma unroll
                    for (int j = 0; j < 3; ++j) N[3 * i + j] = row_dot(R, i, G[j], G[3 + j], G[6 + j]);
                    t[i] = row_dot(R, i, g[0], g[1], g[2]);
                }
            } else {                       // rotation = R_gt R_aug^T
#pragma unroll
                for (int i = 0; i < 3; ++i) {
#pragma unroll
                    for (int j = 0; j < 3; ++j) N[3 * i + j] = row_dot(G, i, R[3 * j], R[3 * j + 1], R[3 * j + 2]);
                    t[i] = g[i];
                }
            }
            if (kitti) {                   // translation = -(R' src_shift) + scale t' + ref_shift
#pragma unroll
                for (int i = 0; i < 3; ++i) t[i] = __dmul_rn(t[i], scale);
                double m[3];
#pragma unroll
                for (int i = 0; i < 3; ++i) m[i] = row_dot(N, i, ss[0], ss[1], ss[2]);
#pragma unroll
                for (int i = 0; i < 3; ++i) t[i] = __dadd_rn(__dadd_rn(-m[i], t[i]), rs[i]);
            }
            float* To = T_out + 16ll * p;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
#pragma unroll
                for (int j = 0; j < 3; ++j) To[4 * i + j] = __double2float_rn(N[3 * i + j]);
                To[4 * i + 3] = __double2float_rn(t[i]);
                To[12 + i] = 0.0f;
            }
            To[15] = 1.0f;
        }
    }
    __syncthreads();
    const int r = blockIdx.x * AUG_POINT_THREADS + threadIdx.x;
    if (r >= Out.count[c]) return;
    const long long o = (long long)Out.start[c] + r;
    const int j = origin[o];
    const float* q = points + 3ll * (In.start[c] + j);
    double x = (double)q[0], y = (double)q[1], z = (double)q[2];
    uint32_t w[4];
    aug_words(w, (uint32_t)j, pair, key, aug_tag(AUG_NOISE, src ? 1u : 0u));
    // numpy: (rand - 0.5) * noise
    const double n0 = __dmul_rn(__dadd_rn(u32(w[0]), -0.5), P.noise);
    const double n1 = __dmul_rn(__dadd_rn(u32(w[1]), -0.5), P.noise);
    const double n2 = __dmul_rn(__dadd_rn(u32(w[2]), -0.5), P.noise);
    const bool rotated = prm[9] != 0.0;
    if (kitti) {                           // noise, rotation, scale, shift
        x = __dadd_rn(x, n0); y = __dadd_rn(y, n1); z = __dadd_rn(z, n2);
        if (rotated) {
            const double a = row_dot(prm, 0, x, y, z), b = row_dot(prm, 1, x, y, z), d = row_dot(prm, 2, x, y, z);
            x = a; y = b; z = d;
        }
        x = __dadd_rn(__dmul_rn(x, prm[10]), prm[11]);
        y = __dadd_rn(__dmul_rn(y, prm[10]), prm[12]);
        z = __dadd_rn(__dmul_rn(z, prm[10]), prm[13]);
    } else {                               // rotation, noise
        if (rotated) {
            const double a = row_dot(prm, 0, x, y, z), b = row_dot(prm, 1, x, y, z), d = row_dot(prm, 2, x, y, z);
            x = a; y = b; z = d;
        }
        x = __dadd_rn(x, n0); y = __dadd_rn(y, n1); z = __dadd_rn(z, n2);
    }
    out[3 * o] = __double2float_rn(x);
    out[3 * o + 1] = __double2float_rn(y);
    out[3 * o + 2] = __double2float_rn(z);
}

// ---- ModelNet ---------------------------------------------------------------------------------------------------------------

// order-preserving map of a double to 64 bits (larger value -> larger key); -0.0 is taken as +0.0
__device__ __forceinline__ unsigned long long ordered_key(double d) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(__dadd_rn(d, 0.0));
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// radix_select_kth over 64-bit keys: MSB-first 8-bit digits, ties at the threshold to the lowest indices (need_eq of them)
template <class Key>
__device__ __forceinline__ void radix_select_kth64(int total, int k, Key key, unsigned* hist, unsigned long long* prefix_s,
                                                   unsigned* kth_s, unsigned long long& thr, int& need_eq) {
    unsigned long long prefix = 0, mask = 0;
    int remaining = k;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (int t = threadIdx.x; t < total; t += blockDim.x) {
            const unsigned long long b = key(t);
            if ((b & mask) == prefix) atomicAdd(&hist[(unsigned)(b >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int rem = remaining;
            int d = 255;
            for (; d > 0; --d) {
                if ((int)hist[d] >= rem) break;
                rem -= (int)hist[d];
            }
            *prefix_s = prefix | ((unsigned long long)d << shift);
            *kth_s = (unsigned)rem;
        }
        __syncthreads();
        prefix = *prefix_s;
        remaining = (int)*kth_s;
        mask |= (255ull << shift);
        __syncthreads();
    }
    thr = prefix;
    need_eq = remaining;
}

struct MnParams {
    int num_points, sort_n;                // sort_n: num_points rounded up to a power of two
    double keep_ratio, rotation_magnitude, translation_magnitude, noise_magnitude;
};

// round(keep N) as the reference's int(floor(N keep + 0.5))
__host__ __device__ __forceinline__ int crop_count(int n, double keep) { return (int)floor((double)n * keep + 0.5); }

// ModelNet pair draws of pair `pair` by one thread: prm = [R (9), t (3), this cloud's plane normal (3)]; the ref cloud also writes
// the record row and the transform.  Not inlined: one thread runs it, and its registers stay out of the kernel's loops.
__device__ __noinline__ void modelnet_draws(const MnParams& P, const AugKey& key, uint32_t pair, int src, double* prm,
                                            double* record, float* T_out) {
        double u[11], R[9];
    pair_uniforms(u, 10, pair, key);
    // numpy: rand(3) * pi * rotation_magnitude / 180; uniform(-m, m) = -m + (m - -m) u
    euler_zyx(__ddiv_rn(__dmul_rn(__dmul_rn(u[0], M_PI), P.rotation_magnitude), 180.0),
              __ddiv_rn(__dmul_rn(__dmul_rn(u[1], M_PI), P.rotation_magnitude), 180.0),
              __ddiv_rn(__dmul_rn(__dmul_rn(u[2], M_PI), P.rotation_magnitude), 180.0), R);
    const double tw = __dsub_rn(P.translation_magnitude, -P.translation_magnitude);
    double t[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] = __dadd_rn(-P.translation_magnitude, __dmul_rn(tw, u[3 + i]));
    // random_sample_plane: phi = uniform(0, 2 pi), theta = uniform(0, pi)
    const double phi = __dmul_rn(__dsub_rn(2.0 * M_PI, 0.0), src ? u[8] : u[6]);
    const double theta = __dmul_rn(__dsub_rn(M_PI, 0.0), src ? u[9] : u[7]);
    double sp, cp, st, ct;
    sincos(phi, &sp, &cp); sincos(theta, &st, &ct);
#pragma unroll
    for (int i = 0; i < 9; ++i) prm[i] = R[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) prm[9 + i] = t[i];
    prm[12] = __dmul_rn(st, cp); prm[13] = __dmul_rn(st, sp); prm[14] = ct;
    if (!src) {
        write_record(record, u, R);
        float* To = T_out;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int j = 0; j < 3; ++j) To[4 * i + j] = __double2float_rn(R[3 * i + j]);
            To[4 * i + 3] = __double2float_rn(t[i]);
            To[12 + i] = 0.0f;
        }
        To[15] = 1.0f;
    }
}

// One CTA per cloud, grid (1, 2B), MN_THREADS; cloud c reads shape c % B.  Dynamic shared memory: the fp64 reduction scratch
// (3 x MN_THREADS), the cropped rows and their sample words (crop_max each), the sort keys (sort_n).  dkey: workspace, the
// distance keys of cloud c at 2 In.start[c % B] + (c >= B) In.count[c % B] + j.
__global__ void __launch_bounds__(MN_THREADS) modelnet_pairs_kernel(
        const float* __restrict__ shapes, const __grid_constant__ Segs In, int B, MnParams P, int crop_max, AugKey key,
        uint32_t pair_base, unsigned long long* __restrict__ dkey, float* __restrict__ out, int* __restrict__ origin,
        float* __restrict__ T_out, double* __restrict__ record) {
    extern __shared__ __align__(16) unsigned char smem[];
    double* red = reinterpret_cast<double*>(smem);
    unsigned long long* sk = reinterpret_cast<unsigned long long*>(red + 3 * MN_THREADS);
    int* crow = reinterpret_cast<int*>(sk + P.sort_n);
    uint32_t* cword = reinterpret_cast<uint32_t*>(crow + crop_max);
    __shared__ double prm[18];             // R (9), t (3), plane normal (3), mean (3)
    __shared__ double inv_scale_s, inv_t[3];
    __shared__ unsigned hist[256];
    __shared__ unsigned long long prefix64_s;
    __shared__ unsigned prefix_s, kth_s;
    __shared__ int warp_tot[MN_THREADS / 32];
    const int c = blockIdx.y, p = c % B, src = c >= B ? 1 : 0;
    const int N = In.count[p], tid = threadIdx.x;
    const float* pts = shapes + 3ll * In.start[p];
    dkey += 2ll * In.start[p] + (long long)src * N;
    const uint32_t pair = pair_base + (uint32_t)p;

    if (tid == 0) modelnet_draws(P, key, pair, src, prm, record + (long long)p * AUG_RECORD, T_out + 16ll * p);
    // 1. normalise: mean in a fixed order (per-thread strided sums, then a tree), then the largest norm
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int j = tid; j < N; j += MN_THREADS) {
        sx = __dadd_rn(sx, (double)pts[3 * j]); sy = __dadd_rn(sy, (double)pts[3 * j + 1]); sz = __dadd_rn(sz, (double)pts[3 * j + 2]);
    }
    red[tid] = sx; red[MN_THREADS + tid] = sy; red[2 * MN_THREADS + tid] = sz;
    __syncthreads();
    for (int s = MN_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
#pragma unroll
            for (int i = 0; i < 3; ++i) red[i * MN_THREADS + tid] = __dadd_rn(red[i * MN_THREADS + tid], red[i * MN_THREADS + tid + s]);
        }
        __syncthreads();
    }
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) prm[15 + i] = __ddiv_rn(red[i * MN_THREADS], (double)N);
    }
    __syncthreads();
    const double mx = prm[15], my = prm[16], mz = prm[17];
    double nmax = 0.0;
    for (int j = tid; j < N; j += MN_THREADS) {
        const double x = __dsub_rn((double)pts[3 * j], mx), y = __dsub_rn((double)pts[3 * j + 1], my), z = __dsub_rn((double)pts[3 * j + 2], mz);
        nmax = fmax(nmax, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z))));
    }
    red[tid] = nmax;
    __syncthreads();
    for (int s = MN_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) red[tid] = fmax(red[tid], red[tid + s]);
        __syncthreads();
    }
    if (tid == 0) inv_scale_s = red[0];
    __syncthreads();
    const double scale = inv_scale_s;
    // 2. the cloud's point j: normalised, and for src the image under the inverse transform (p R + (-R^T t)); R, t and the
    //    inverse translation are read from shared memory
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) inv_t[i] = -col_dot(prm, i, prm[9], prm[10], prm[11]);
    }
    __syncthreads();
    auto point = [&](int j, double& x, double& y, double& z) {
        x = __ddiv_rn(__dsub_rn((double)pts[3 * j], mx), scale);
        y = __ddiv_rn(__dsub_rn((double)pts[3 * j + 1], my), scale);
        z = __ddiv_rn(__dsub_rn((double)pts[3 * j + 2], mz), scale);
        if (src) {
            const double a = __dadd_rn(col_dot(prm, 0, x, y, z), inv_t[0]);
            const double b = __dadd_rn(col_dot(prm, 1, x, y, z), inv_t[1]);
            const double d = __dadd_rn(col_dot(prm, 2, x, y, z), inv_t[2]);
            x = a; y = b; z = d;
        }
    };
    // 3. plane distances
    const double n0 = prm[12], n1 = prm[13], n2 = prm[14];
    for (int j = tid; j < N; j += MN_THREADS) {
        double x, y, z;
        point(j, x, y, z);
        dkey[j] = ordered_key(__dadd_rn(__dadd_rn(__dmul_rn(x, n0), __dmul_rn(y, n1)), __dmul_rn(z, n2)));
    }
    __syncthreads();
    // 4. crop: the K largest distances, ties to the lowest row, in ascending row with their sample words
    const int K = crop_count(N, P.keep_ratio);
    unsigned long long thr64;
    int need_eq;
    radix_select_kth64(N, K, [&](int j) { return dkey[j]; }, hist, &prefix64_s, &kth_s, thr64, need_eq);
    {
        int kept = 0, eq = 0;
        for (int base = 0; base < N; base += MN_THREADS) {
            const int j = base + tid;
            const unsigned long long b = j < N ? dkey[j] : 0ull;
            const bool fe = j < N && b == thr64;
            int te;
            const int re = chunk_rank<MN_THREADS / 32>(fe, warp_tot, &te);
            const bool f = j < N && (b > thr64 || (fe && eq + re < need_eq));
            int tot;
            const int r = chunk_rank<MN_THREADS / 32>(f, warp_tot, &tot);
            if (f) {
                uint32_t w[4];
                aug_words(w, (uint32_t)j, pair, key, aug_tag(AUG_SAMPLE, (uint32_t)src));
                crow[kept + r] = j;
                cword[kept + r] = w[0];
            }
            kept += tot; eq += te;
        }
    }
    __syncthreads();
    // 5. sample and shuffle: the num_points smallest keys (word << 32) | row, in key order
    const int M = P.num_points;
    if (K > M) {
        unsigned thr;
        int ne;
        radix_select_kth((long long)K, M, [&](long long i) { return ~cword[i]; }, hist, &prefix_s, &kth_s, thr, ne);
        int kept = 0, eq = 0;
        for (int base = 0; base < K; base += MN_THREADS) {
            const int i = base + tid;
            const unsigned b = i < K ? ~cword[i] : 0u;
            const bool fe = i < K && b == thr;
            int te;
            const int re = chunk_rank<MN_THREADS / 32>(fe, warp_tot, &te);
            const bool f = i < K && (b > thr || (fe && eq + re < ne));
            int tot;
            const int r = chunk_rank<MN_THREADS / 32>(f, warp_tot, &tot);
            if (f) sk[kept + r] = ((unsigned long long)cword[i] << 32) | (unsigned)crow[i];
            kept += tot; eq += te;
        }
    } else {
        for (int i = tid; i < K; i += MN_THREADS) sk[i] = ((unsigned long long)cword[i] << 32) | (unsigned)crow[i];
    }
    for (int i = M + tid; i < P.sort_n; i += MN_THREADS) sk[i] = ~0ull;
    __syncthreads();
    for (int k = 2; k <= P.sort_n; k <<= 1) {              // bitonic sort, ascending
        for (int h = k >> 1; h > 0; h >>= 1) {
            for (int i = tid; i < P.sort_n; i += MN_THREADS) {
                const int l = i ^ h;
                if (l > i) {
                    const unsigned long long a = sk[i], b = sk[l];
                    if ((a > b) == ((i & k) == 0)) { sk[i] = b; sk[l] = a; }
                }
            }
            __syncthreads();
        }
    }
    // 6. jitter: clip(0.01 N(0, 1), +-noise_magnitude) by Box-Muller from the row's words, one rounding to fp32
    const long long o0 = (long long)c * M;
    for (int r = tid; r < M; r += MN_THREADS) {
        const int j = (int)(unsigned)(sk[r] & 0xFFFFFFFFull);
        double x, y, z;
        point(j, x, y, z);
        uint32_t w[4];
        aug_words(w, (uint32_t)j, pair, key, aug_tag(AUG_JITTER, (uint32_t)src));
        const double r0 = sqrt(-2.0 * log(__dsub_rn(1.0, u32(w[0])))), r1 = sqrt(-2.0 * log(__dsub_rn(1.0, u32(w[2]))));
        double s0, c0, s1, c1;
        sincos(__dmul_rn(2.0 * M_PI, u32(w[1])), &s0, &c0);
        sincos(__dmul_rn(2.0 * M_PI, u32(w[3])), &s1, &c1);
        const double m = P.noise_magnitude;
        const double jx = fmin(fmax(__dmul_rn(0.01, __dmul_rn(r0, c0)), -m), m);
        const double jy = fmin(fmax(__dmul_rn(0.01, __dmul_rn(r0, s0)), -m), m);
        const double jz = fmin(fmax(__dmul_rn(0.01, __dmul_rn(r1, c1)), -m), m);
        origin[o0 + r] = j;
        out[3 * (o0 + r)] = __double2float_rn(__dadd_rn(x, jx));
        out[3 * (o0 + r) + 1] = __double2float_rn(__dadd_rn(y, jy));
        out[3 * (o0 + r) + 2] = __double2float_rn(__dadd_rn(z, jz));
    }
}

// ---- ModelNet validation / test pairs (deterministic) -------------------------------------------------------------------------

constexpr int MNB_THREADS = 256;
constexpr int MNB_MAX_PAIRS = 1024;        // pairs per launch; the entry point splits larger calls

struct MnbPair {
    long long start;                       // first row of the shape in `shapes`
    int count;                             // its points
    uint32_t index;                        // the dataset index, which seeds the pair's stream
};

// scipy's Rotation.from_euler('zyx', (a, b, c)).as_matrix() in scipy's own arithmetic: elementary quaternions (axis sin(angle / 2),
// cos(angle / 2)), composed extrinsically q = qx(c) (qy(b) qz(a)) without normalisation, then the matrix of q.  euler_zyx's
// direct product is the same rotation but not the same bits.
__device__ __forceinline__ void quat_compose(const double (&p)[4], const double (&q)[4], double (&r)[4]) {
    const double c0 = __dsub_rn(__dmul_rn(p[1], q[2]), __dmul_rn(p[2], q[1]));
    const double c1 = __dsub_rn(__dmul_rn(p[2], q[0]), __dmul_rn(p[0], q[2]));
    const double c2 = __dsub_rn(__dmul_rn(p[0], q[1]), __dmul_rn(p[1], q[0]));
    r[0] = __dadd_rn(__dadd_rn(__dmul_rn(p[3], q[0]), __dmul_rn(q[3], p[0])), c0);
    r[1] = __dadd_rn(__dadd_rn(__dmul_rn(p[3], q[1]), __dmul_rn(q[3], p[1])), c1);
    r[2] = __dadd_rn(__dadd_rn(__dmul_rn(p[3], q[2]), __dmul_rn(q[3], p[2])), c2);
    r[3] = __dsub_rn(__dmul_rn(p[3], q[3]),
                     __dadd_rn(__dadd_rn(__dmul_rn(p[0], q[0]), __dmul_rn(p[1], q[1])), __dmul_rn(p[2], q[2])));
}

// sin x and cos x correctly rounded for |x| <= 1.6 (the half-angles of Euler angles within +-pi, with margin): Horner's form of the
// Taylor series in double-double, sin x = x (1 - x^2 / (2 3) (1 - x^2 / (4 5) (...))) and cos x = 1 - x^2 / (1 2) (1 - ...), 18
// terms each (the first omitted term is below 2^-120 of the result), with every operation rounded explicitly (no contraction).
// The double-double result is within about 2^-100 relative, so its rounding to double is the correctly rounded value unless the
// exact value lies that close to a midpoint.  The device's sincos may be an ulp off; the host libm's (which scipy calls) is
// correctly rounded except in rare near-tie cases.
struct DD {
    double hi, lo;
};
__device__ __forceinline__ DD dd_norm(double a, double b) {          // fast two-sum, |a| >= |b|
    const double s = __dadd_rn(a, b);
    return DD{s, __dsub_rn(b, __dsub_rn(s, a))};
}
__device__ __forceinline__ DD dd_mul(DD a, DD b) {
    const double p = __dmul_rn(a.hi, b.hi);
    const double e = __fma_rn(a.hi, b.hi, -p);
    return dd_norm(p, __dadd_rn(e, __dadd_rn(__dmul_rn(a.hi, b.lo), __dmul_rn(a.lo, b.hi))));
}
__device__ __forceinline__ DD dd_div(DD a, double d) {               // a / d for an exact integer d
    const double q = __ddiv_rn(a.hi, d);
    const double r = __dadd_rn(__fma_rn(-q, d, a.hi), a.lo);
    return dd_norm(q, __ddiv_rn(r, d));
}
__device__ __forceinline__ DD dd_one_minus(DD a) {                   // 1 - a
    const double s = __dsub_rn(1.0, a.hi);
    const double bb = __dsub_rn(s, 1.0);
    const double e = __dadd_rn(__dsub_rn(1.0, __dsub_rn(s, bb)), __dsub_rn(-a.hi, bb));      // two-sum error of 1 + (-a.hi)
    return dd_norm(s, __dsub_rn(e, a.lo));
}
__device__ __forceinline__ void sincos_cr(double x, double* s, double* c) {
    const double p = __dmul_rn(x, x);
    const DD x2 = dd_norm(p, __fma_rn(x, x, -p));
    DD ts{1.0, 0.0}, tc{1.0, 0.0};
#pragma unroll 1
    for (int k = 18; k >= 1; --k) {
        ts = dd_one_minus(dd_div(dd_mul(ts, x2), (double)((2 * k) * (2 * k + 1))));
        tc = dd_one_minus(dd_div(dd_mul(tc, x2), (double)((2 * k - 1) * (2 * k))));
    }
    const double sp = __dmul_rn(x, ts.hi);
    *s = __dadd_rn(sp, __dadd_rn(__fma_rn(x, ts.hi, -sp), __dmul_rn(x, ts.lo)));
    *c = __dadd_rn(tc.hi, tc.lo);
}

// CR: the half-angles' sin and cos correctly rounded (sincos_cr; the rotated 3DMatch pairs), else the device's sincos (the ModelNet
// pairs, unchanged)
template <bool CR = false>
__device__ __forceinline__ void euler_zyx_scipy(double a, double b, double c, double (&R)[9]) {
    double qz[4] = {0.0, 0.0, 0.0, 0.0}, qy[4] = {0.0, 0.0, 0.0, 0.0}, qx[4] = {0.0, 0.0, 0.0, 0.0}, t[4], q[4];
    if constexpr (CR) {
        sincos_cr(__dmul_rn(a, 0.5), &qz[2], &qz[3]);
        sincos_cr(__dmul_rn(b, 0.5), &qy[1], &qy[3]);
        sincos_cr(__dmul_rn(c, 0.5), &qx[0], &qx[3]);
    } else {
        sincos(__dmul_rn(a, 0.5), &qz[2], &qz[3]);
        sincos(__dmul_rn(b, 0.5), &qy[1], &qy[3]);
        sincos(__dmul_rn(c, 0.5), &qx[0], &qx[3]);
    }
    quat_compose(qy, qz, t);
    quat_compose(qx, t, q);
    const double x2 = __dmul_rn(q[0], q[0]), y2 = __dmul_rn(q[1], q[1]), z2 = __dmul_rn(q[2], q[2]), w2 = __dmul_rn(q[3], q[3]);
    const double xy = __dmul_rn(q[0], q[1]), zw = __dmul_rn(q[2], q[3]), xz = __dmul_rn(q[0], q[2]);
    const double yw = __dmul_rn(q[1], q[3]), yz = __dmul_rn(q[1], q[2]), xw = __dmul_rn(q[0], q[3]);
    R[0] = __dadd_rn(__dsub_rn(__dsub_rn(x2, y2), z2), w2);
    R[1] = __dmul_rn(2.0, __dsub_rn(xy, zw));
    R[2] = __dmul_rn(2.0, __dadd_rn(xz, yw));
    R[3] = __dmul_rn(2.0, __dadd_rn(xy, zw));
    R[4] = __dadd_rn(__dsub_rn(__dadd_rn(-x2, y2), z2), w2);
    R[5] = __dmul_rn(2.0, __dsub_rn(yz, xw));
    R[6] = __dmul_rn(2.0, __dsub_rn(xz, yw));
    R[7] = __dmul_rn(2.0, __dadd_rn(yz, xw));
    R[8] = __dadd_rn(__dadd_rn(__dsub_rn(-x2, y2), z2), w2);
}

// The permutation(n) of the stream (arange, then for i = n-1 .. 1 swap i with interval(i)) left in perm[0 .. n); lane 0 swaps.
__device__ __forceinline__ void legacy_permutation(LegacyRandom& rng, int* perm, int n) {
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < n; i += 32) perm[i] = i;
    __syncwarp();
    for (int i = n - 1; i > 0; --i) {
        const int j = (int)rng.interval((uint32_t)i);
        if (lane == 0) {
            const int a = perm[i];
            perm[i] = perm[j];
            perm[j] = a;
        }
    }
    __syncwarp();
}

// Every draw of one pair, in the reference's order, by the whole of warp 0 (warp-uniform): prm = [R (9), t (3), ref plane normal
// (3), src plane normal (3), inverse translation -(R^T t) (3)]; sel (2 x M): the sampled positions in each cloud's crop order
// (random_sample_points, padding included); shuf (2 x M): each cloud's final shuffle; jit (6 M, global): the clipped jitter of
// ref then src in the order drawn; scratch: K words.
__device__ __forceinline__ void mnb_draws(uint32_t index, int K, const MnParams& P, uint32_t* mt, double* prm, int* scratch, int* sel,
                                       int* shuf, double* jit, float* T_out) {
    const int lane = threadIdx.x & 31, M = P.num_points;
    LegacyRandom rng{mt, 0, false, 0.0};
    rng.seed(index);
    // random_sample_transform: rand(3) pi magnitude / 180, Rotation.from_euler('zyx'); uniform(-m, m, 3)
    double e[3], t[3], R[9];
#pragma unroll
    for (int i = 0; i < 3; ++i) e[i] = __ddiv_rn(__dmul_rn(__dmul_rn(rng.next_double(), M_PI), P.rotation_magnitude), 180.0);
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] = rng.uniform(-P.translation_magnitude, P.translation_magnitude);
    euler_zyx_scipy(e[0], e[1], e[2], R);
    // random_sample_plane of ref, then of src: phi = uniform(0, 2 pi), theta = uniform(0, pi)
    double nrm[6];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const double phi = rng.uniform(0.0, 2.0 * M_PI), theta = rng.uniform(0.0, M_PI);
        double sp, cp, st, ct;
        sincos(phi, &sp, &cp); sincos(theta, &st, &ct);
        nrm[3 * c] = __dmul_rn(st, cp); nrm[3 * c + 1] = __dmul_rn(st, sp); nrm[3 * c + 2] = ct;
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < 9; ++i) prm[i] = R[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) prm[9 + i] = t[i];
#pragma unroll
        for (int i = 0; i < 6; ++i) prm[12 + i] = nrm[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) prm[18 + i] = -col_dot(R, i, t[0], t[1], t[2]);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int j = 0; j < 3; ++j) T_out[4 * i + j] = __double2float_rn(R[3 * i + j]);
            T_out[4 * i + 3] = __double2float_rn(t[i]);
            T_out[12 + i] = 0.0f;
        }
        T_out[15] = 1.0f;
    }
    // random_sample_points of ref, then of src: the first M of permutation(K), or the permutation repeated and its head
    for (int c = 0; c < 2; ++c) {
        legacy_permutation(rng, scratch, K);
        for (int r = lane; r < M; r += 32) sel[c * M + r] = scratch[r % K];
        __syncwarp();
    }
    // random_jitter_points of ref, then of src: clip(0 + 0.01 gauss, +-noise_magnitude); the Gaussian cached by the last ref draw
    // (3 M odd) is the first of src
    for (int k = 0; k < 6 * M; ++k) {
        const double g = fmin(fmax(__dadd_rn(0.0, __dmul_rn(0.01, rng.gauss_draw())), -P.noise_magnitude), P.noise_magnitude);
        if (lane == 0) jit[k] = g;
    }
    // random_shuffle_points of ref, then of src
    legacy_permutation(rng, shuf, M);
    legacy_permutation(rng, shuf + M, M);
}

// normalize_points in fp32, by one warp: the column sums in row order, / N, to mean[3]; then the largest sqrt((x^2 + y^2) + z^2)
// of the centred points to *scale.  The normalised coordinate is normalized(v, mean, scale).  The benchmark pairs and the raw
// shapes share these two, so a pair's points and its raw_points come from the same normalisation.
__device__ __forceinline__ void normalize_stats(const float* __restrict__ pts, int N, float* mean, float* scale) {
    const int lane = threadIdx.x & 31;
    if (lane < 3) {
        float s = 0.0f;
        for (int j = 0; j < N; ++j) s = __fadd_rn(s, pts[3 * j + lane]);
        mean[lane] = __fdiv_rn(s, (float)N);
    }
    __syncwarp();
    const float mx = mean[0], my = mean[1], mz = mean[2];
    float nmax = 0.0f;
    for (int j = lane; j < N; j += 32) {
        const float x = __fsub_rn(pts[3 * j], mx), y = __fsub_rn(pts[3 * j + 1], my), z = __fsub_rn(pts[3 * j + 2], mz);
        nmax = fmaxf(nmax, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = fmaxf(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    if (lane == 0) *scale = nmax;
}

__device__ __forceinline__ float normalized(float v, float mean, float scale) { return __fdiv_rn(__fsub_rn(v, mean), scale); }

// The ModelNet item's raw_points: normalize_points(shape) in fp32.  One CTA per shape, grid (n, 1), MNB_THREADS: warp 0 takes the
// statistics, then the CTA writes the rows.  The output has the input's layout.
__global__ void __launch_bounds__(MNB_THREADS) modelnet_raw_kernel(const float* __restrict__ shapes, const MnbPair* __restrict__ pairs,
                                                                   float* __restrict__ out) {
    __shared__ float mean_s[3], scale_s;
    const MnbPair pr = pairs[blockIdx.x];
    const float* pts = shapes + 3ll * pr.start;
    if (threadIdx.x < 32) normalize_stats(pts, pr.count, mean_s, &scale_s);
    __syncthreads();
    const float scale = scale_s;
    float* o = out + 3ll * pr.start;
    for (int i = threadIdx.x; i < 3 * pr.count; i += MNB_THREADS) o[i] = normalized(pts[i], mean_s[i % 3], scale);
}

// One CTA per pair, grid (n, 1), MNB_THREADS.  Warp 0 consumes the pair's stream (mnb_draws) while warp 1 normalises the shape in
// fp32; then the CTA orders each cloud's crop (bitonic sort of (distance desc, row asc)), maps the samples to shape rows, and writes
// the jittered, shuffled points.  Dynamic shared memory: sort keys and rows (sort_n each; the draws' scratch aliases them), sel and
// shuf (2 M each).  jit: workspace, 6 M doubles per pair of the launch.
__global__ void __launch_bounds__(MNB_THREADS) modelnet_benchmark_kernel(
        const float* __restrict__ shapes, const MnbPair* __restrict__ pairs, int total_pairs, int pair0, MnParams P,
        double* __restrict__ jit_ws, float* __restrict__ out, int* __restrict__ origin, float* __restrict__ T_out) {
    extern __shared__ __align__(16) unsigned char smem[];
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(smem);
    int* srow = reinterpret_cast<int*>(skey + P.sort_n);
    int* sel = srow + P.sort_n;
    int* shuf = sel + 2 * P.num_points;
    __shared__ uint32_t mt[MT_N];
    __shared__ double prm[21];
    __shared__ float mean_s[3], scale_s;
    const int q = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, M = P.num_points;
    const MnbPair pr = pairs[q];
    const int N = pr.count, K = crop_count(N, P.keep_ratio);
    const float* pts = shapes + 3ll * pr.start;
    double* jit = jit_ws + 6ll * M * q;

    if (warp == 0) {
        mnb_draws(pr.index, K, P, mt, prm, reinterpret_cast<int*>(skey), sel, shuf, jit, T_out + 16ll * (pair0 + q));
    } else if (warp == 1) {
        normalize_stats(pts, N, mean_s, &scale_s);
    }
    __syncthreads();
    const float mx = mean_s[0], my = mean_s[1], mz = mean_s[2], scale = scale_s;
    // point j of cloud c: the normalised fp32 point, and for src its image p R + (-(R^T t)) in fp64
    auto point = [&](int c, int j, double& x, double& y, double& z) {
        x = (double)normalized(pts[3 * j], mx, scale);
        y = (double)normalized(pts[3 * j + 1], my, scale);
        z = (double)normalized(pts[3 * j + 2], mz, scale);
        if (c) {
            const double a = __dadd_rn(col_dot(prm, 0, x, y, z), prm[18]);
            const double b = __dadd_rn(col_dot(prm, 1, x, y, z), prm[19]);
            const double d = __dadd_rn(col_dot(prm, 2, x, y, z), prm[20]);
            x = a; y = b; z = d;
        }
    };
    for (int c = 0; c < 2; ++c) {
        // random_crop_point_cloud_with_plane: rows by descending (x nx + y ny) + z nz, ties to the lowest row; sorted ascending on
        // (~ordered_key(d), row)
        const double n0 = prm[12 + 3 * c], n1 = prm[13 + 3 * c], n2 = prm[14 + 3 * c];
        for (int j = tid; j < P.sort_n; j += MNB_THREADS) {
            unsigned long long k = ~0ull;
            if (j < N) {
                double x, y, z;
                point(c, j, x, y, z);
                k = ~ordered_key(__dadd_rn(__dadd_rn(__dmul_rn(x, n0), __dmul_rn(y, n1)), __dmul_rn(z, n2)));
            }
            skey[j] = k;
            srow[j] = j < N ? j : 0x7fffffff;
        }
        __syncthreads();
        for (int k = 2; k <= P.sort_n; k <<= 1) {          // bitonic sort, ascending
            for (int h = k >> 1; h > 0; h >>= 1) {
                for (int i = tid; i < P.sort_n; i += MNB_THREADS) {
                    const int l = i ^ h;
                    if (l > i) {
                        const unsigned long long a = skey[i], b = skey[l];
                        const int ra = srow[i], rb = srow[l];
                        const bool gt = a > b || (a == b && ra > rb);
                        if (gt == ((i & k) == 0)) { skey[i] = b; skey[l] = a; srow[i] = rb; srow[l] = ra; }
                    }
                }
                __syncthreads();
            }
        }
        // crop position -> shape row
        for (int r = tid; r < M; r += MNB_THREADS) sel[c * M + r] = srow[sel[c * M + r]];
        __syncthreads();
    }
    // jitter, shuffle, round to fp32: output s of cloud c is sample shuf[s] of that cloud
    for (int i = tid; i < 2 * M; i += MNB_THREADS) {
        const int c = i >= M ? 1 : 0, s = i - c * M, k = shuf[c * M + s], row = sel[c * M + k];
        double x, y, z;
        point(c, row, x, y, z);
        const double* g = jit + 3ll * (c * M + k);
        const long long o = ((long long)c * total_pairs + pair0 + q) * M + s;
        origin[o] = row;
        out[3 * o] = __double2float_rn(__dadd_rn(x, g[0]));
        out[3 * o + 1] = __double2float_rn(__dadd_rn(y, g[1]));
        out[3 * o + 2] = __double2float_rn(__dadd_rn(z, g[2]));
    }
}

// ---- Rotated 3DMatch / 3DLoMatch benchmark pairs ------------------------------------------------------------------------------

constexpr int ROT_MAX_PAIRS = 64;          // pairs per launch; the entry point splits larger calls
constexpr int ROT_THREADS = 256;

// One launch's pairs, by value: its clouds are ref clouds 0 .. n-1 then src clouds 0 .. n-1, rows start[c] .. start[c+1] - 1 of the
// launch; the ref rows begin at row ref_row0 of the call's stack and the src rows at src_row0.
struct RotLaunch {
    int n, pair0;
    long long ref_row0, src_row0;
    long long start[2 * ROT_MAX_PAIRS + 1];
    uint32_t index[ROT_MAX_PAIRS];
};

// random_sample_rotation_v2: axis = rand(3) - 0.5; axis = axis / norm(axis) + 1e-8; theta = pi rand(); R = from_euler('zyx',
// axis theta).  numpy's norm of three doubles is sqrt(dot), and OpenBLAS's dot is the FMA chain below.
__device__ __forceinline__ void rotation_v2(LegacyRandom& rng, double (&R)[9]) {
    double a[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) a[i] = __dsub_rn(rng.next_double(), 0.5);
    const double norm = __dsqrt_rn(__fma_rn(a[2], a[2], __fma_rn(a[1], a[1], __dmul_rn(a[0], a[0]))));
    const double theta = __dmul_rn(M_PI, rng.next_double());
    double e[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) e[i] = __dmul_rn(__dadd_rn(__ddiv_rn(a[i], norm), 1e-8), theta);
    euler_zyx_scipy<true>(e[0], e[1], e[2], R);
}

// numpy's 3 x 3 products in OpenBLAS's order: C = A B with A B[i, j] = fma(a2, b2, fma(a1, b1, a0 b0)) over row i of A and column
// j of B (B_T: B is given transposed), and A v = fma(a2, v2, fma(a0, v0, a1 v1)) (dgemv)
__device__ __forceinline__ double dot3_gemm(double a0, double a1, double a2, double b0, double b1, double b2) {
    return __fma_rn(a2, b2, __fma_rn(a1, b1, __dmul_rn(a0, b0)));
}

// One warp per pair, grid (n): draws R_ref then R_src from np.random.seed(index) and composes the pair's transform in fp64:
// rotation = R_ref rotation R_src^T, translation = R_ref translation; rounds it to fp32 once.
__global__ void __launch_bounds__(32) rotated_draws_kernel(RotLaunch Lc, const double* __restrict__ T_in, float* __restrict__ T_out,
                                                           double* __restrict__ rot) {
    __shared__ uint32_t mt[MT_N];
    const int q = blockIdx.x, p = Lc.pair0 + q;
    LegacyRandom rng{mt, 0, false, 0.0};
    rng.seed(Lc.index[q]);
    double Rr[9], Rs[9];
    rotation_v2(rng, Rr);
    rotation_v2(rng, Rs);
    if (threadIdx.x != 0) return;
    const double* T = T_in + 16ll * p;
    double A[9], t[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) A[3 * i + j] = dot3_gemm(Rr[3 * i], Rr[3 * i + 1], Rr[3 * i + 2], T[j], T[4 + j], T[8 + j]);
        t[i] = __fma_rn(Rr[3 * i + 2], T[11], __fma_rn(Rr[3 * i], T[3], __dmul_rn(Rr[3 * i + 1], T[7])));
    }
    float* o = T_out + 16ll * p;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) o[4 * i + j] = __double2float_rn(dot3_gemm(A[3 * i], A[3 * i + 1], A[3 * i + 2], Rs[3 * j], Rs[3 * j + 1], Rs[3 * j + 2]));
        o[4 * i + 3] = __double2float_rn(t[i]);
        o[12 + i] = 0.0f;
    }
    o[15] = 1.0f;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        rot[18ll * p + i] = Rr[i];
        rot[18ll * p + 9 + i] = Rs[i];
    }
}

// One thread per row of the launch: p R^T in fp64 in numpy's (N, 3) x (3, 3) order, fma(z, R[i,2], fma(y, R[i,1], x R[i,0])), rounded
// to fp32 once.
// Real: the clouds' type as the dataset files hold them (fp32 widens exactly).
template <typename Real>
__global__ void __launch_bounds__(ROT_THREADS) rotated_points_kernel(RotLaunch Lc, const Real* __restrict__ pts, const double* __restrict__ rot,
                                                                     float* __restrict__ out) {
    const long long r = (long long)blockIdx.x * ROT_THREADS + threadIdx.x;
    const int nc = 2 * Lc.n;
    if (r >= Lc.start[nc]) return;
    int lo = 0, hi = nc - 1;                 // the cloud c with start[c] <= r < start[c + 1]
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (Lc.start[mid] <= r) lo = mid;
        else hi = mid - 1;
    }
    const int c = lo, src = c >= Lc.n;
    const long long row = src ? Lc.src_row0 + (r - Lc.start[Lc.n]) : Lc.ref_row0 + r;
    const double* R = rot + 18ll * (Lc.pair0 + c - (src ? Lc.n : 0)) + 9 * src;
    const double x = (double)pts[3 * row], y = (double)pts[3 * row + 1], z = (double)pts[3 * row + 2];
#pragma unroll
    for (int i = 0; i < 3; ++i) out[3 * row + i] = __double2float_rn(dot3_gemm(x, y, z, R[3 * i], R[3 * i + 1], R[3 * i + 2]));
}

static int next_pow2(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

static AugKey make_key(uint64_t seed, uint64_t iteration) {
    return AugKey{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)iteration, (uint32_t)(iteration >> 32)};
}

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_augment_pairs_batched_workspace_bytes(int64_t n_rows) {
    return align_up(4 * (size_t)(n_rows > 0 ? n_rows : 0), 256) + 256;
}

int geob200_augment_pairs_batched(const float* points, const int64_t* lengths_h, int64_t n_pairs, const float* transforms, int mode,
                                  int64_t point_limit, double noise, double rotation_factor, double min_scale, double max_scale,
                                  double shift, uint64_t seed, uint64_t iteration, int64_t pair_base, float* out_points, int32_t* origin,
                                  float* out_transforms, double* record, void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "augment_pairs_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(mode == GEOB200_AUGMENT_3DMATCH || mode == GEOB200_AUGMENT_KITTI, "augment_pairs_batched: unknown mode %d", mode);
    GEOB_REQUIRE(point_limit > 0 && point_limit < (1ll << 31), "augment_pairs_batched: point_limit must be in 1..2^31-1");
    GEOB_REQUIRE(isfinite(noise) && noise >= 0.0, "augment_pairs_batched: noise must be finite and non-negative");
    GEOB_REQUIRE(isfinite(rotation_factor) && rotation_factor > 0.0, "augment_pairs_batched: rotation_factor must be finite and positive");
    GEOB_REQUIRE(isfinite(min_scale) && isfinite(max_scale) && min_scale <= max_scale,
                 "augment_pairs_batched: scales must be finite with min_scale <= max_scale");
    GEOB_REQUIRE(isfinite(shift) && shift >= 0.0, "augment_pairs_batched: shift must be finite and non-negative");
    GEOB_REQUIRE(pair_base >= 0 && pair_base + n_pairs <= 0xFFFFFFFFll, "augment_pairs_batched: pair_base out of range");
    GEOB_REQUIRE(lengths_h != nullptr, "augment_pairs_batched: null lengths");
    GEOB_REQUIRE(points != nullptr && transforms != nullptr && out_points != nullptr && origin != nullptr && out_transforms != nullptr &&
                     record != nullptr,
                 "augment_pairs_batched: null pointer");
    const int B = (int)n_pairs;
    int64_t kept[GEOB_MAX_CLOUDS];
    for (int c = 0; c < 2 * B; ++c) {
        GEOB_REQUIRE(lengths_h[c] > 0, "augment_pairs_batched: cloud %d is empty", c);
        kept[c] = lengths_h[c] < point_limit ? lengths_h[c] : point_limit;
    }
    Segs In, Out;
    if (segs_from_counts(&In, 2 * B, lengths_h) || segs_from_counts(&Out, 2 * B, kept)) return -1;
    const int64_t rows = (int64_t)In.start[2 * B - 1] + In.count[2 * B - 1];
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_augment_pairs_batched_workspace_bytes(rows),
                 "augment_pairs_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    uint32_t* word = ar.take<uint32_t>((size_t)rows);
    GEOB_REQUIRE(ar.ok(), "augment_pairs_batched: workspace accounting error");
    cudaStream_t st = (cudaStream_t)stream;
    const AugKey key = make_key(seed, iteration);
    point_limit_kernel<<<dim3(1, 2 * B), AUG_THREADS, 0, st>>>(In, Out, B, (int)point_limit, key, (uint32_t)pair_base, word, origin);
    GEOB_CHECK_LAUNCH();
    const AugParams P{mode, noise, rotation_factor, min_scale, max_scale, shift};
    const unsigned gx = (unsigned)((Out.max + AUG_POINT_THREADS - 1) / AUG_POINT_THREADS);
    augment_points_kernel<<<dim3(gx, 2 * B), AUG_POINT_THREADS, 0, st>>>(points, In, Out, origin, transforms, B, P, key, (uint32_t)pair_base,
                                                                       out_points, out_transforms, record);
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

size_t geob200_modelnet_pairs_batched_workspace_bytes(int64_t n_rows) {
    return align_up(16 * (size_t)(n_rows > 0 ? n_rows : 0), 256) + 256;
}

int geob200_modelnet_pairs_batched(const float* shapes, const int64_t* lengths_h, int64_t n_pairs, int64_t num_points, double keep_ratio,
                                   double rotation_magnitude, double translation_magnitude, double noise_magnitude, uint64_t seed,
                                   uint64_t iteration, int64_t pair_base, float* out_points, int32_t* origin, float* out_transforms,
                                   double* record, void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && 2 * n_pairs <= GEOB_MAX_CLOUDS, "modelnet_pairs_batched: 1..%d pairs", GEOB_MAX_CLOUDS / 2);
    GEOB_REQUIRE(num_points > 0 && num_points <= MN_MAX_POINTS, "modelnet_pairs_batched: num_points must be in 1..%d", MN_MAX_POINTS);
    GEOB_REQUIRE(isfinite(keep_ratio) && keep_ratio > 0.0 && keep_ratio <= 1.0, "modelnet_pairs_batched: keep_ratio must be in (0, 1]");
    GEOB_REQUIRE(isfinite(rotation_magnitude) && isfinite(translation_magnitude) && isfinite(noise_magnitude) &&
                     rotation_magnitude >= 0.0 && translation_magnitude >= 0.0 && noise_magnitude >= 0.0,
                 "modelnet_pairs_batched: magnitudes must be finite and non-negative");
    GEOB_REQUIRE(pair_base >= 0 && pair_base + n_pairs <= 0xFFFFFFFFll, "modelnet_pairs_batched: pair_base out of range");
    GEOB_REQUIRE(lengths_h != nullptr, "modelnet_pairs_batched: null lengths");
    GEOB_REQUIRE(shapes != nullptr && out_points != nullptr && origin != nullptr && out_transforms != nullptr && record != nullptr,
                 "modelnet_pairs_batched: null pointer");
    const int B = (int)n_pairs;
    int crop_max = 0;
    for (int p = 0; p < B; ++p) {
        GEOB_REQUIRE(lengths_h[p] > 0 && lengths_h[p] <= MN_MAX_SHAPE, "modelnet_pairs_batched: shape %d has %lld points (1..%d)", p,
                     (long long)lengths_h[p], MN_MAX_SHAPE);
        const int K = crop_count((int)lengths_h[p], keep_ratio);
        GEOB_REQUIRE(K >= num_points, "modelnet_pairs_batched: shape %d keeps round(%g * %lld) = %d < num_points = %lld points", p,
                     keep_ratio, (long long)lengths_h[p], K, (long long)num_points);
        crop_max = K > crop_max ? K : crop_max;
    }
    Segs In;
    if (segs_from_counts(&In, B, lengths_h)) return -1;
    const int64_t rows = (int64_t)In.start[B - 1] + In.count[B - 1];
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_modelnet_pairs_batched_workspace_bytes(rows),
                 "modelnet_pairs_batched: workspace too small");
    Arena ar(workspace, workspace_bytes);
    unsigned long long* dkey = ar.take<unsigned long long>(2 * (size_t)rows);
    GEOB_REQUIRE(ar.ok(), "modelnet_pairs_batched: workspace accounting error");
    MnParams P{(int)num_points, next_pow2((int)num_points), keep_ratio, rotation_magnitude, translation_magnitude, noise_magnitude};
    const size_t smem = 3 * MN_THREADS * sizeof(double) + (size_t)P.sort_n * 8 + (size_t)crop_max * 8;
    if (smem > 48 * 1024 && ensure_max_smem((const void*)modelnet_pairs_kernel)) return -1;
    modelnet_pairs_kernel<<<dim3(1, 2 * B), MN_THREADS, smem, (cudaStream_t)stream>>>(shapes, In, B, P, crop_max, make_key(seed, iteration),
                                                                                     (uint32_t)pair_base, dkey, out_points, origin,
                                                                                     out_transforms, record);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

size_t geob200_modelnet_benchmark_pairs_batched_workspace_bytes(int64_t n_pairs, int64_t num_points) {
    const size_t b = (size_t)(n_pairs < 1 ? 0 : n_pairs < MNB_MAX_PAIRS ? n_pairs : MNB_MAX_PAIRS);
    const size_t m = (size_t)(num_points > 0 ? num_points : 0);
    return align_up(b * sizeof(MnbPair), 256) + align_up(b * 6 * m * sizeof(double), 256) + 256;
}

int geob200_modelnet_benchmark_pairs_batched(const float* shapes, const int64_t* lengths_h, const int64_t* indices_h, int64_t n_pairs,
                                             int64_t num_points, double keep_ratio, double rotation_magnitude, double translation_magnitude,
                                             double noise_magnitude, float* out_points, int32_t* origin, float* out_transforms,
                                             void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs < (1ll << 31) / MN_MAX_POINTS / 2, "modelnet_benchmark_pairs_batched: n_pairs must be in 1..%lld",
                 (1ll << 31) / MN_MAX_POINTS / 2 - 1);
    GEOB_REQUIRE(num_points > 0 && num_points <= MN_MAX_POINTS, "modelnet_benchmark_pairs_batched: num_points must be in 1..%d",
                 MN_MAX_POINTS);
    GEOB_REQUIRE(isfinite(keep_ratio) && keep_ratio > 0.0 && keep_ratio <= 1.0,
                 "modelnet_benchmark_pairs_batched: keep_ratio must be in (0, 1]");
    GEOB_REQUIRE(isfinite(rotation_magnitude) && isfinite(translation_magnitude) && isfinite(noise_magnitude) &&
                     rotation_magnitude >= 0.0 && translation_magnitude >= 0.0 && noise_magnitude >= 0.0,
                 "modelnet_benchmark_pairs_batched: magnitudes must be finite and non-negative");
    GEOB_REQUIRE(lengths_h != nullptr && indices_h != nullptr, "modelnet_benchmark_pairs_batched: null lengths or indices");
    GEOB_REQUIRE(shapes != nullptr && out_points != nullptr && origin != nullptr && out_transforms != nullptr,
                 "modelnet_benchmark_pairs_batched: null pointer");
    for (int64_t p = 0; p < n_pairs; ++p) {
        GEOB_REQUIRE(lengths_h[p] > 0 && lengths_h[p] <= MN_MAX_SHAPE, "modelnet_benchmark_pairs_batched: shape %lld has %lld points (1..%d)",
                     (long long)p, (long long)lengths_h[p], MN_MAX_SHAPE);
        GEOB_REQUIRE(crop_count((int)lengths_h[p], keep_ratio) >= 1, "modelnet_benchmark_pairs_batched: shape %lld keeps no point",
                     (long long)p);
        GEOB_REQUIRE(indices_h[p] >= 0 && indices_h[p] <= 0xFFFFFFFFll, "modelnet_benchmark_pairs_batched: index %lld of pair %lld is "
                     "not in 0..2^32-1", (long long)indices_h[p], (long long)p);
    }
    GEOB_REQUIRE(workspace != nullptr &&
                     workspace_bytes >= geob200_modelnet_benchmark_pairs_batched_workspace_bytes(n_pairs, num_points),
                 "modelnet_benchmark_pairs_batched: workspace too small");
    const int B = (int)n_pairs, M = (int)num_points;
    const int cap = B < MNB_MAX_PAIRS ? B : MNB_MAX_PAIRS;
    Arena ar(workspace, workspace_bytes);
    MnbPair* table = ar.take<MnbPair>((size_t)cap);
    double* jit = ar.take<double>((size_t)cap * 6 * M);
    GEOB_REQUIRE(ar.ok(), "modelnet_benchmark_pairs_batched: workspace accounting error");
    cudaStream_t st = (cudaStream_t)stream;
    MnbPair host[MNB_MAX_PAIRS];
    long long start = 0;
    int launches = 0;
    for (int p0 = 0; p0 < B; p0 += cap) {
        const int n = B - p0 < cap ? B - p0 : cap;
        int nmax = 1;
        for (int q = 0; q < n; ++q) {
            host[q] = MnbPair{start, (int)lengths_h[p0 + q], (uint32_t)indices_h[p0 + q]};
            start += lengths_h[p0 + q];
            nmax = host[q].count > nmax ? host[q].count : nmax;
        }
        // from pageable memory: staged before the call returns, ordered before the launch on the stream
        GEOB_CHECK_CUDA(cudaMemcpyAsync(table, host, (size_t)n * sizeof(MnbPair), cudaMemcpyHostToDevice, st));
        const MnParams P{M, next_pow2(nmax), keep_ratio, rotation_magnitude, translation_magnitude, noise_magnitude};
        const size_t smem = (size_t)P.sort_n * (sizeof(unsigned long long) + sizeof(int)) + (size_t)4 * M * sizeof(int);
        if (smem > 48 * 1024 && ensure_max_smem((const void*)modelnet_benchmark_kernel)) return -1;
        modelnet_benchmark_kernel<<<n, MNB_THREADS, smem, st>>>(shapes, table, B, p0, P, jit, out_points, origin, out_transforms);
        GEOB_CHECK_LAUNCH();
        ++launches;
    }
    count_launches(launches);
    return 0;
}

size_t geob200_modelnet_raw_points_batched_workspace_bytes(int64_t n_shapes) {
    const size_t b = (size_t)(n_shapes < 1 ? 0 : n_shapes < MNB_MAX_PAIRS ? n_shapes : MNB_MAX_PAIRS);
    return align_up(b * sizeof(MnbPair), 256) + 256;
}

int geob200_modelnet_raw_points_batched(const float* shapes, const int64_t* lengths_h, int64_t n_shapes, float* out_points,
                                        void* workspace, size_t workspace_bytes, void* stream) {
    GEOB_REQUIRE(n_shapes > 0 && n_shapes < (1ll << 31) / MN_MAX_SHAPE, "modelnet_raw_points_batched: n_shapes must be in 1..%lld",
                 (1ll << 31) / MN_MAX_SHAPE - 1);
    GEOB_REQUIRE(lengths_h != nullptr, "modelnet_raw_points_batched: null lengths");
    GEOB_REQUIRE(shapes != nullptr && out_points != nullptr, "modelnet_raw_points_batched: null pointer");
    for (int64_t p = 0; p < n_shapes; ++p)
        GEOB_REQUIRE(lengths_h[p] > 0 && lengths_h[p] <= MN_MAX_SHAPE, "modelnet_raw_points_batched: shape %lld has %lld points (1..%d)",
                     (long long)p, (long long)lengths_h[p], MN_MAX_SHAPE);
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_modelnet_raw_points_batched_workspace_bytes(n_shapes),
                 "modelnet_raw_points_batched: workspace too small");
    const int B = (int)n_shapes;
    const int cap = B < MNB_MAX_PAIRS ? B : MNB_MAX_PAIRS;
    Arena ar(workspace, workspace_bytes);
    MnbPair* table = ar.take<MnbPair>((size_t)cap);
    GEOB_REQUIRE(ar.ok(), "modelnet_raw_points_batched: workspace accounting error");
    cudaStream_t st = (cudaStream_t)stream;
    MnbPair host[MNB_MAX_PAIRS];
    long long start = 0;
    int launches = 0;
    for (int p0 = 0; p0 < B; p0 += cap) {
        const int n = B - p0 < cap ? B - p0 : cap;
        for (int q = 0; q < n; ++q) {
            host[q] = MnbPair{start, (int)lengths_h[p0 + q], 0u};
            start += lengths_h[p0 + q];
        }
        // from pageable memory: staged before the call returns, ordered before the launch on the stream
        GEOB_CHECK_CUDA(cudaMemcpyAsync(table, host, (size_t)n * sizeof(MnbPair), cudaMemcpyHostToDevice, st));
        modelnet_raw_kernel<<<n, MNB_THREADS, 0, st>>>(shapes, table, out_points);
        GEOB_CHECK_LAUNCH();
        ++launches;
    }
    count_launches(launches);
    return 0;
}

int geob200_rotated_pairs_batched(const void* points, int points_fp64, const int64_t* lengths_h, const int64_t* indices_h, int64_t n_pairs,
                                  const double* transforms, float* out_points, float* out_transforms, double* rotations, void* stream) {
    GEOB_REQUIRE(n_pairs > 0 && n_pairs <= (1ll << 30), "rotated_pairs_batched: n_pairs must be in 1..2^30");
    GEOB_REQUIRE(points_fp64 == 0 || points_fp64 == 1, "rotated_pairs_batched: points_fp64 must be 0 or 1");
    GEOB_REQUIRE(lengths_h != nullptr && indices_h != nullptr, "rotated_pairs_batched: null lengths or indices");
    GEOB_REQUIRE(points != nullptr && transforms != nullptr && out_points != nullptr && out_transforms != nullptr && rotations != nullptr,
                 "rotated_pairs_batched: null pointer");
    long long rows = 0;
    for (int64_t c = 0; c < 2 * n_pairs; ++c) {
        GEOB_REQUIRE(lengths_h[c] > 0 && lengths_h[c] < (1ll << 31), "rotated_pairs_batched: cloud %lld has %lld points (1..2^31-1)",
                     (long long)c, (long long)lengths_h[c]);
        rows += lengths_h[c];
        GEOB_REQUIRE(rows < (1ll << 31), "rotated_pairs_batched: more than 2^31-1 rows in all");
    }
    for (int64_t p = 0; p < n_pairs; ++p)
        GEOB_REQUIRE(indices_h[p] >= 0 && indices_h[p] <= 0xFFFFFFFFll, "rotated_pairs_batched: index %lld of pair %lld is not in "
                     "0..2^32-1", (long long)indices_h[p], (long long)p);
    const int B = (int)n_pairs;
    cudaStream_t st = (cudaStream_t)stream;
    long long ref_row = 0, src_row = 0;
    for (int p = 0; p < B; ++p) src_row += lengths_h[p];
    int launches = 0;
    for (int p0 = 0; p0 < B; p0 += ROT_MAX_PAIRS) {
        RotLaunch Lc;
        Lc.n = B - p0 < ROT_MAX_PAIRS ? B - p0 : ROT_MAX_PAIRS;
        Lc.pair0 = p0;
        Lc.ref_row0 = ref_row;
        Lc.src_row0 = src_row;
        long long s = 0;
        for (int c = 0; c < 2 * Lc.n; ++c) {
            Lc.start[c] = s;
            s += lengths_h[c < Lc.n ? p0 + c : B + p0 + c - Lc.n];
        }
        Lc.start[2 * Lc.n] = s;
        for (int q = 0; q < Lc.n; ++q) {
            Lc.index[q] = (uint32_t)indices_h[p0 + q];
            ref_row += lengths_h[p0 + q];
            src_row += lengths_h[B + p0 + q];
        }
        rotated_draws_kernel<<<Lc.n, 32, 0, st>>>(Lc, transforms, out_transforms, rotations);
        GEOB_CHECK_LAUNCH();
        const unsigned grid = (unsigned)((s + ROT_THREADS - 1) / ROT_THREADS);
        if (points_fp64)
            rotated_points_kernel<<<grid, ROT_THREADS, 0, st>>>(Lc, (const double*)points, rotations, out_points);
        else
            rotated_points_kernel<<<grid, ROT_THREADS, 0, st>>>(Lc, (const float*)points, rotations, out_points);
        GEOB_CHECK_LAUNCH();
        launches += 2;
    }
    count_launches(launches);
    return 0;
}

}  // extern "C"
