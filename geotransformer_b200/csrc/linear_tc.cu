// nn.Linear on the Hopper tensor cores (wgmma): Y[M,N] = X[M,K] . W[N,K]^T + b (optional ReLU), fp32 in / fp32 out.
//
// The reference's Linears are true fp32 (torch default allow_tf32=False), so the product is computed with the
// error-compensated 3xTF32 scheme: x = x_hi + x_lo, w = w_hi + w_lo (hi = top 19 bits), D += x_hi w_hi + x_hi w_lo +
// x_lo w_hi with fp32 accumulation (~1e-6 relative, same as an fp32 FMA chain).
//
// One 128 x BN output tile at a time (BN = min(N,128)), K in chunks of 32 floats (one 128-byte swizzle row); a CTA walks the
// tiles t = blockIdx.x, blockIdx.x + gridDim.x, ... (one tile per CTA unless the persistent loop is on), 384 threads:
//   warps 0-7   consumers    : two warpgroups, rows [0,64) and [64,128) of the tile: wgmma.m64n{BN}k8 tf32, 3 per K-step,
//                              main products and corrections in two register accumulators; then the epilogue straight from
//                              the registers (row scale, bias, ReLU, stores, optional GroupNorm statistics)
//   warp 8      TMA producer : cp.async.bulk.tensor.2d of the raw X tile (128 x 32) and W tile (BN x 32) through SWIZZLE_128B
//                              tensor maps; out-of-bounds rows/columns are zero-filled by the TMA unit
//   warps 9-11  splitters    : in-place hi = tf32_rn(x), lo = x - hi into a second buffer (generic proxy ->
//                              fence.proxy.async), so the MMA sees exact tf32 operands
// The operand ring runs across tile boundaries: the producer and splitters prepare the next tile while the consumers store.
#include <cuda.h>

#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "geob200.h"
#include "hopper.cuh"

namespace geob200 {
namespace ltc {

using namespace hop;

constexpr int BM = 128;
constexpr int KC = 32;
constexpr int TILE_A = BM * 128;       // 16 KB
constexpr int TILE_B = 128 * 128;      // 16 KB (BN <= 128 rows)
constexpr int STAGE = 2 * TILE_A + 2 * TILE_B;   // raw/hi + lo for both operands = 64 KB
constexpr int NSTAGE = 3;
constexpr int PRODUCER_WARP = 8;
constexpr int NSPLIT_WARPS = 3;                       // warps 9..11
constexpr int NTHREADS = (PRODUCER_WARP + 1 + NSPLIT_WARPS) * 32;   // 384
// operand stages + barriers + GroupNorm column sums [8 warps][128] float2 + the bias row, after 1024-byte alignment slack
constexpr int SMEM = NSTAGE * STAGE + 1024 + 256 + 8 * 128 * 8 + 512;

// splitter: in-place hi = tf32_rn(x), lo = x - hi into the second buffer of each operand (element-wise, so the swizzled
// positions are irrelevant: same offset in the hi and lo buffers).  Two 16-byte vectors per thread and iteration: their
// shared-memory round trips overlap.  t = thread index among the NSPLIT_WARPS * 32 splitter threads.
__device__ __forceinline__ void split_stage(unsigned char* st, int BN, int t) {
    constexpr int NT = NSPLIT_WARPS * 32;
    const int nvec_a = TILE_A / 16, nvec_b = BN * 128 / 16;
    const int nvec = nvec_a + nvec_b;
    for (int v0 = t; v0 < nvec; v0 += 2 * NT) {
        const int v1 = v0 + NT;
        unsigned char* p0 = (v0 < nvec_a) ? (st + v0 * 16) : (st + 2 * TILE_A + (v0 - nvec_a) * 16);
        unsigned char* l0 = p0 + ((v0 < nvec_a) ? TILE_A : TILE_B);
        const bool two = v1 < nvec;
        unsigned char* p1 = !two ? p0 : (v1 < nvec_a) ? (st + v1 * 16) : (st + 2 * TILE_A + (v1 - nvec_a) * 16);
        unsigned char* l1 = p1 + ((v1 < nvec_a) ? TILE_A : TILE_B);
        const float4 x0 = *reinterpret_cast<float4*>(p0);
        const float4 x1 = *reinterpret_cast<float4*>(p1);
        float4 h0, q0, h1, q1;
        h0.x = tf32_rn(x0.x); q0.x = x0.x - h0.x;     // round-to-nearest split: |lo| <= 2^-12 |x|, unbiased
        h0.y = tf32_rn(x0.y); q0.y = x0.y - h0.y;
        h0.z = tf32_rn(x0.z); q0.z = x0.z - h0.z;
        h0.w = tf32_rn(x0.w); q0.w = x0.w - h0.w;
        h1.x = tf32_rn(x1.x); q1.x = x1.x - h1.x;
        h1.y = tf32_rn(x1.y); q1.y = x1.y - h1.y;
        h1.z = tf32_rn(x1.z); q1.z = x1.z - h1.z;
        h1.w = tf32_rn(x1.w); q1.w = x1.w - h1.w;
        *reinterpret_cast<float4*>(p0) = h0;
        *reinterpret_cast<float4*>(l0) = q0;
        if (two) {
            *reinterpret_cast<float4*>(p1) = h1;
            *reinterpret_cast<float4*>(l1) = q1;
        }
    }
    fence_proxy_async();
}

// BNI = wgmma N (32, 64 or 128) >= BN; B rows [BN, BNI) of a stage hold stale data and only feed output columns that are
// never stored.  Tile t -> (split z, row tile, column tile), column tile fastest: neighbouring CTAs share their X rows in L2.
template <int BNI>
__global__ void __launch_bounds__(NTHREADS, 1) linear_tc_kernel(const __grid_constant__ CUtensorMap map_x,
                                                                const __grid_constant__ CUtensorMap map_w,
                                                                const float* __restrict__ bias, const float* __restrict__ row_scale,
                                                                float* __restrict__ Y, int ldy, int M, int N, int K, int BN, int relu,
                                                                GnFuse gn, float* __restrict__ splitk_out, int chunks_per_split,
                                                                int col_tiles, int row_tiles, int num_tiles) {
    constexpr int R = BNI / 2;          // accumulator registers per thread
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = (uint64_t*)(smem + NSTAGE * STAGE);
    uint64_t* raw_full = bars;                  // TMA landed
    uint64_t* split_full = bars + NSTAGE;       // hi/lo ready
    uint64_t* empty = bars + 2 * NSTAGE;        // MMAs done with the stage
    float2* gn_sm = (float2*)(smem + NSTAGE * STAGE + 256);        // [8 consumer warps][128 columns] (sum, sum of squares)
    float* bias_s = (float*)(gn_sm + 8 * 128);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nk = (K + KC - 1) / KC;
    const int tiles_per_split = col_tiles * row_tiles;

    if (threadIdx.x == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&split_full[s], NSPLIT_WARPS); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const int z = t / tiles_per_split, rem = t % tiles_per_split;
                const int m0 = (rem / col_tiles) * BM, n0 = (rem % col_tiles) * BN;
                const int kc0 = z * chunks_per_split, kc1 = min(nk, kc0 + chunks_per_split);
                for (int kc = kc0; kc < kc1; ++kc) {
                    mbar_wait(&empty[s], ph ^ 1u);
                    unsigned char* st = smem + s * STAGE;
                    mbar_arrive_expect_tx(&raw_full[s], (uint32_t)(TILE_A + BN * 128));
                    tma_load_2d(st, &map_x, kc * KC, m0, &raw_full[s]);
                    tma_load_2d(st + 2 * TILE_A, &map_w, kc * KC, n0, &raw_full[s]);
                    if (++s == NSTAGE) { s = 0; ph ^= 1u; }
                }
            }
        }
        return;
    }
    if (warp > PRODUCER_WARP) {
        const int ts = threadIdx.x - (PRODUCER_WARP + 1) * 32;
        int s = 0;
        uint32_t ph = 0;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            const int z = t / tiles_per_split;
            const int kc0 = z * chunks_per_split, kc1 = min(nk, kc0 + chunks_per_split);
            for (int kc = kc0; kc < kc1; ++kc) {
                mbar_wait(&raw_full[s], ph);
                split_stage(smem + s * STAGE, BN, ts);
                __syncwarp();
                if (lane == 0) mbar_arrive(&split_full[s]);
                if (++s == NSTAGE) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ---- consumers ----
    const int wg = warp >> 2, wq = warp & 3;
    int s = 0;
    uint32_t ph = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int z = t / tiles_per_split, rem = t % tiles_per_split;
        const int ty = rem / col_tiles;
        const int m0 = ty * BM, n0 = (rem % col_tiles) * BN;
        const int kc0 = z * chunks_per_split, kc1 = min(nk, kc0 + chunks_per_split);
        // the tile's bias row goes through shared memory once: per-element global loads in the epilogue would be a chain of
        // dependent L2 round trips
        asm volatile("bar.sync 1, 256;" ::: "memory");                          // previous tile's readers of bias_s / gn_sm are done
        if (threadIdx.x < 128) bias_s[threadIdx.x] = (bias != nullptr && (int)threadIdx.x < BN) ? __ldg(bias + n0 + threadIdx.x) : 0.f;
        asm volatile("bar.sync 1, 256;" ::: "memory");

        // main products and the (2^-11 smaller) correction products go to separate accumulators: keeping the number of
        // additions into the main accumulator at K/8 instead of 3K/8 lowers the rounding error of the fp32 accumulation
        float acc[R], cor[R];
#pragma unroll
        for (int i = 0; i < R; ++i) { acc[i] = 0.f; cor[i] = 0.f; }
        int prev_s = -1;
        for (int kc = kc0; kc < kc1; ++kc) {
            mbar_wait(&split_full[s], ph);
            const uint32_t st = smem_u32(smem + s * STAGE);
            const uint64_t a_hi = make_desc(st + wg * (TILE_A / 2)), a_lo = make_desc(st + TILE_A + wg * (TILE_A / 2));
            const uint64_t b_hi = make_desc(st + 2 * TILE_A), b_lo = make_desc(st + 2 * TILE_A + TILE_B);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < KC / 8; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);      // +32 bytes in 16-byte units
                const uint32_t accum = (kc == kc0 && kk == 0) ? 0u : 1u;
                wgmma_tf32<BNI>(acc, a_hi + adv, b_hi + adv, accum);
                wgmma_tf32<BNI>(cor, a_hi + adv, b_lo + adv, accum);
                wgmma_tf32<BNI>(cor, a_lo + adv, b_hi + adv, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();                    // the previous chunk's MMAs are done: its stage can be refilled
            if (prev_s >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev_s]); }
            prev_s = s;
            if (++s == NSTAGE) { s = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
        reg_fence(acc);
        reg_fence(cor);
        if (prev_s >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev_s]); }

        // epilogue: this thread holds rows r0 and r0 + 8, columns 8j + 2(lane % 4) + {0, 1}
        const int r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
        const int c0 = 2 * (lane & 3);
        float rs[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) rs[h] = (row_scale != nullptr && r0 + 8 * h < M) ? row_scale[r0 + 8 * h] : 1.0f;
        if (splitk_out != nullptr) {              // raw partial sums of this K-slice (N is even: float2-aligned)
#pragma unroll
            for (int j = 0; j < BNI / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = r0 + 8 * h, col = 8 * j + c0;
                    if (m < M && col < BN)
                        *reinterpret_cast<float2*>(splitk_out + ((long long)z * M + m) * N + n0 + col) =
                            make_float2(acc[4 * j + 2 * h] + cor[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + cor[4 * j + 2 * h + 1]);
                }
            continue;
        }
        const bool vec2 = ((ldy & 1) == 0) && ((reinterpret_cast<uintptr_t>(Y) & 7) == 0);
#pragma unroll
        for (int j = 0; j < BNI / 8; ++j) {
            const int col = 8 * j + c0;
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float v = (acc[4 * j + e] + cor[4 * j + e]) * rs[e >> 1] + bias_s[col + (e & 1)];
                if (relu) v = fmaxf(v, 0.f);
                o[e] = v;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = r0 + 8 * h;
                if (m < M && col < BN) {
                    float* yp = Y + (long long)m * ldy + n0 + col;
                    if (vec2) *reinterpret_cast<float2*>(yp) = make_float2(o[2 * h], o[2 * h + 1]);
                    else { yp[0] = o[2 * h]; yp[1] = o[2 * h + 1]; }
                }
            }
            if (gn.groups > 0) {
                // column sums over the warp's 16 rows (rows past M and columns past BN contribute nothing)
                const bool ok0 = r0 < M && col < BN, ok1 = r0 + 8 < M && col < BN;
                float a0 = (ok0 ? o[0] : 0.f) + (ok1 ? o[2] : 0.f), a1 = (ok0 ? o[1] : 0.f) + (ok1 ? o[3] : 0.f);
                float q0 = (ok0 ? o[0] * o[0] : 0.f) + (ok1 ? o[2] * o[2] : 0.f);
                float q1 = (ok0 ? o[1] * o[1] : 0.f) + (ok1 ? o[3] * o[3] : 0.f);
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
                    a0 += __shfl_xor_sync(0xffffffffu, a0, off);
                    a1 += __shfl_xor_sync(0xffffffffu, a1, off);
                    q0 += __shfl_xor_sync(0xffffffffu, q0, off);
                    q1 += __shfl_xor_sync(0xffffffffu, q1, off);
                }
                if (lane < 4) {
                    gn_sm[warp * 128 + col] = make_float2(a0, q0);
                    gn_sm[warp * 128 + col + 1] = make_float2(a1, q1);
                }
            }
        }
        if (gn.groups > 0) {
            // per-tile partial in a fixed order; gn_finalize / gn_seg_finalize (kpconv.cu) fold the tiles afterwards
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const int sw = gn.slot_width, slots_tile = BN / sw, slots_total = N / sw;
            const int et = threadIdx.x;
            if (et < slots_tile) {
                double s1 = 0.0, s2 = 0.0;
                for (int w = 0; w < 8; ++w) {
                    float f1 = 0.f, f2 = 0.f;
                    for (int c = 0; c < sw; ++c) {
                        const float2 p = gn_sm[w * 128 + et * sw + c];
                        f1 += p.x;
                        f2 += p.y;
                    }
                    s1 += (double)f1;
                    s2 += (double)f2;
                }
                double* dst = gn.partial + ((long long)ty * slots_total + n0 / sw + et) * 2;
                dst[0] = s1;
                dst[1] = s2;
            }
        }
    }
}

// y[m][n] = (sum_z P[z][m][n]) * row_scale[m] + bias[n] (+ ReLU): the splits are added in a fixed order
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ P, int splits, long long MN, int N,
                                                            const float* __restrict__ bias, const float* __restrict__ row_scale,
                                                            float* __restrict__ Y, int ldy, int relu) {
    const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i4 >= MN) return;
    float4 a = *reinterpret_cast<const float4*>(P + i4);
    for (int z = 1; z < splits; ++z) {
        const float4 b = *reinterpret_cast<const float4*>(P + (long long)z * MN + i4);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    const long long m = i4 / N;
    const int n = (int)(i4 % N);
    const float rs = row_scale != nullptr ? row_scale[m] : 1.0f;
    float o[4] = {a.x * rs, a.y * rs, a.z * rs, a.w * rs};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        if (bias != nullptr) o[u] += bias[n + u];
        if (relu) o[u] = fmaxf(o[u], 0.f);
    }
    float* y = Y + m * ldy + n;
    if ((reinterpret_cast<uintptr_t>(y) & 15) == 0) *reinterpret_cast<float4*>(y) = make_float4(o[0], o[1], o[2], o[3]);
    else { y[0] = o[0]; y[1] = o[1]; y[2] = o[2]; y[3] = o[3]; }
}

// cuTensorMapEncodeTiled is fetched through the runtime (cudaGetDriverEntryPoint) so that libgeob200.so does not link
// libcuda directly and still loads on a machine without a driver (the no-GPU ABI tests).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

static int encode_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (fn == nullptr) { set_error("cuTensorMapEncodeTiled entry point not available"); return -1; }
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return -1; }
    return 0;
}

}  // namespace ltc

// ---- optional per-launch profile (bench.py roofline): CUDA events around every linear_tc launch + its shape ----------------
struct ProfRec { cudaEvent_t a, b; long long m, n, k; };
static std::vector<ProfRec> g_prof;
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static bool g_splitk_on = true;
static bool g_persistent_on = true;    // persistent tile loop for GEMMs of more than one wave of tiles (geob200_set_linear_persistent)

// ---- split-K scratch: one grow-only buffer per stream (like a BLAS workspace; freed with the process) ---------------------
struct SplitWs { void* ptr; size_t bytes; };
static std::vector<std::pair<cudaStream_t, SplitWs>> g_split_ws;
static std::mutex g_split_mu;
static float* splitk_scratch(cudaStream_t st, size_t bytes) {
    std::lock_guard<std::mutex> lk(g_split_mu);
    for (auto& e : g_split_ws)
        if (e.first == st) {
            if (e.second.bytes >= bytes) return (float*)e.second.ptr;
            // stream-ordered free: earlier kernels on this stream may still read the old buffer
            cudaFreeAsync(e.second.ptr, st);
            e.second = {nullptr, 0};
            if (cudaMallocAsync(&e.second.ptr, bytes * 2, st) != cudaSuccess) return nullptr;
            e.second.bytes = bytes * 2;
            return (float*)e.second.ptr;
        }
    SplitWs w{nullptr, 0};
    const size_t cap = bytes * 2 > (16u << 20) ? bytes * 2 : (16u << 20);
    if (cudaMallocAsync(&w.ptr, cap, st) != cudaSuccess) return nullptr;
    w.bytes = cap;
    g_split_ws.push_back({st, w});
    return (float*)w.ptr;
}

// returns 1 when the shape/alignment is not handled by the tensor-core path (caller falls back to the fp32 kernel)
int linear_tc(const float* x, int64_t ldx, const float* w, int64_t ldw, const float* bias, const float* row_scale, float* y, int64_t ldy,
              int64_t m, int64_t n, int64_t k, int relu, cudaStream_t st, const GnFuse* gn) {
    if (m < 64 || n < 32 || (n % 16) != 0 || (k % 4) != 0 || (ldx % 4) != 0 || (ldw % 4) != 0) return 1;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15)) return 1;
    if (n > 128 && (n % 128) != 0) return 1;
    const int BN = (int)(n >= 128 ? 128 : n);
    CUtensorMap mx, mw;
    if (ltc::encode_map(&mx, x, m, k, ldx, ltc::BM)) return -1;
    if (ltc::encode_map(&mw, w, n, k, ldw, BN)) return -1;
    const int col_tiles = (int)(n / BN), row_tiles = (int)((m + ltc::BM - 1) / ltc::BM);
    GnFuse g{};
    if (gn != nullptr) {
        g = *gn;
        const int64_t cpg = n / g.groups;
        // groups must tile the 32-column epilogue chunks: cpg in {1,2,4,...,32} or a multiple of 32 dividing the column tile
        if (g.groups <= 0 || n % g.groups != 0 || (cpg < 32 ? (32 % cpg) != 0 : (cpg % 32) != 0 || (BN % cpg) != 0) || relu) return 1;
        g.slot_width = (int)(cpg < 32 ? cpg : 32);
    }
    // split-K: a deep K loop on a handful of tiles leaves most SMs idle and is pure latency (1.4 us per 32-wide chunk): give
    // every K-slice of >= 8 chunks its own CTA when the grid would cover less than half of the GPU
    const int nk = (int)((k + ltc::KC - 1) / ltc::KC);
    const int tiles = col_tiles * row_tiles;
    int splits = 1;
    if (g_splitk_on && tiles * 2 <= num_sms() && nk >= 16) {
        splits = nk / 8;
        if (splits > num_sms() / tiles) splits = num_sms() / tiles;
        if (splits > 16) splits = 16;
        if (splits < 2) splits = 1;
    }
    // the epilogue statistics need the complete sums: with split-K the caller runs the stand-alone GroupNorm statistics instead
    if (gn != nullptr && splits > 1) return 1;
    int cps = nk;
    float* part = nullptr;
    if (splits > 1) {
        cps = (nk + splits - 1) / splits;
        splits = (nk + cps - 1) / cps;
        part = splitk_scratch(st, (size_t)splits * (size_t)m * (size_t)n * sizeof(float));
        if (part == nullptr) { splits = 1; cps = nk; }
    }
    ProfRec rec{};
    const bool prof = g_prof_on;
    if (prof) {
        cudaEventCreate(&rec.a);
        cudaEventCreate(&rec.b);
        rec.m = m; rec.n = n; rec.k = k;
        cudaEventRecord(rec.a, st);
    }
    // one CTA per tile, or (persistent loop) one CTA per SM walking the tiles of a GEMM of more than one wave
    const int num_tiles = tiles * splits;
    const bool persistent = g_persistent_on && splits == 1 && tiles > num_sms();
    const unsigned grid = (unsigned)(persistent ? num_sms() : num_tiles);
    const void* kern = BN <= 32 ? (const void*)ltc::linear_tc_kernel<32> : BN <= 64 ? (const void*)ltc::linear_tc_kernel<64>
                                                                                      : (const void*)ltc::linear_tc_kernel<128>;
    if (ensure_max_smem(kern)) return -1;
#define GEOB_LTC_LAUNCH(BNI)                                                                                                  \
    ltc::linear_tc_kernel<BNI><<<grid, ltc::NTHREADS, ltc::SMEM, st>>>(mx, mw, bias, row_scale, y, (int)ldy, (int)m, (int)n, (int)k, \
                                                                       BN, relu, g, part, cps, col_tiles, row_tiles, num_tiles)
    if (BN <= 32) GEOB_LTC_LAUNCH(32);
    else if (BN <= 64) GEOB_LTC_LAUNCH(64);
    else GEOB_LTC_LAUNCH(128);
#undef GEOB_LTC_LAUNCH
    if (part != nullptr) {
        const long long mn = (long long)m * n;
        ltc::splitk_reduce_kernel<<<(unsigned)((mn / 4 + 255) / 256), 256, 0, st>>>(part, splits, mn, (int)n, bias, row_scale, y, (int)ldy, relu);
        count_launches(1);
    }
    if (prof) {
        cudaEventRecord(rec.b, st);
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_prof.push_back(rec);
    }
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // namespace geob200

extern "C" {

int geob200_set_linear_persistent(int on) {
    geob200::g_persistent_on = on != 0;
    return 0;
}

int geob200_set_split_k(int on) {
    geob200::g_splitk_on = on != 0;
    return 0;
}

// Profiling aid for bench.py: while enabled every tensor-core GEMM launch is bracketed by CUDA events on its stream.
int geob200_linear_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(geob200::g_prof_mu);
    for (auto& r : geob200::g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    geob200::g_prof.clear();
    geob200::g_prof_on = on != 0;
    return 0;
}

// Synchronises the recorded launches and returns their number; shapes[3*i..] = (m, n, k), ms[i] = kernel time.
int64_t geob200_linear_profile_read(int64_t capacity, int64_t* shapes, float* ms) {
    std::lock_guard<std::mutex> lk(geob200::g_prof_mu);
    int64_t n = 0;
    for (auto& r : geob200::g_prof) {
        if (n >= capacity) break;
        if (cudaEventSynchronize(r.b) != cudaSuccess) break;
        float t = 0.f;
        cudaEventElapsedTime(&t, r.a, r.b);
        shapes[3 * n] = r.m; shapes[3 * n + 1] = r.n; shapes[3 * n + 2] = r.k;
        ms[n] = t;
        ++n;
    }
    return n;
}

}  // extern "C"
