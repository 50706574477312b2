// nn.Linear on the Hopper tensor cores (wgmma): Y[M,N] = X[M,K] . W[N,K]^T + b (optional ReLU), fp32 in / fp32 out.
//
// The reference's Linears are true fp32 (torch default allow_tf32=False), so the product is computed with the
// error-compensated 3xTF32 scheme: x = x_hi + x_lo, w = w_hi + w_lo (hi = top 19 bits), D += x_hi w_hi + x_hi w_lo +
// x_lo w_hi with fp32 accumulation (~1e-6 relative, same as an fp32 FMA chain).
//
// The weight is split once, outside the GEMM, into a tf32 image [W_hi (N x K) | W_lo (N x K)] (geob200_split_tf32); the
// activations are split in registers where they are consumed.
//
// One 128 x BN output tile at a time (BN = min(N,128)), K in chunks of 32 floats (one 128-byte swizzle row); a CTA walks the
// tiles t = blockIdx.x, blockIdx.x + gridDim.x, ... (one tile per CTA unless the persistent loop is on), 384 threads:
//   warps 0-7   consumers    : two warpgroups, rows [0,64) and [64,128) of the tile.  Per 8-wide K-step each thread loads its
//                              A fragment from the raw fp32 X tile, splits it (hi = tf32_rn(x), lo = x - hi) and issues
//                              wgmma.m64n{BN}k8 tf32 with A from registers, 3 per K-step, main products and corrections in
//                              two register accumulators; then the epilogue straight from the registers (row scale, bias,
//                              ReLU, stores, optional GroupNorm statistics)
//   warps 8-11  producer     : one thread of warp 8 issues cp.async.bulk.tensor.2d of the X tile (128 x 32) and of the W_hi
//                              and W_lo tiles (BN x 32 each, two loads through one map of the 2N x K image) through
//                              SWIZZLE_128B tensor maps; out-of-bounds rows/columns are zero-filled by the TMA unit
// The producer is a whole warpgroup only so that setmaxnreg can move its registers to the consumers (which hold a chunk's 32
// A fragment registers besides the 2 x BN/2 accumulator registers): 4 x 32 x 40 + 8 x 32 x 232 <= 65536.
// The operand ring runs across tile boundaries: the producer loads the next tile while the consumers store.
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
constexpr int STAGE = TILE_A + 2 * TILE_B;       // raw X + W_hi + W_lo = 48 KB
constexpr int NSTAGE = 4;
constexpr int PRODUCER_WARP = 8;
constexpr int NTHREADS = (PRODUCER_WARP + 4) * 32;   // 384
// operand stages + barriers + GroupNorm column sums [8 warps][128] float2 + the bias row, after 1024-byte alignment slack
constexpr int SMEM = NSTAGE * STAGE + 1024 + 256 + 8 * 128 * 8 + 512;

// [hi | lo] image of a row-major (n x k, leading dimension ld) fp32 matrix: out[r][c] = tf32_rn(w), out[n + r][c] = w - hi
__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ w, long long ld, long long n, long long k,
                                                         float* __restrict__ out) {
    const long long nk = n * k;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nk; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / k, c = i % k;
        const float x = w[r * ld + c];
        const float hi = tf32_rn(x);
        out[i] = hi;
        out[nk + i] = x - hi;
    }
}

// BNI = wgmma N (32, 64 or 128) >= BN; B rows [BN, BNI) of a stage hold stale data and only feed output columns that are
// never stored.  Tile t -> (split z, row tile, column tile), column tile fastest: neighbouring CTAs share their X rows in L2.
// map_w covers the 2N x K weight image: W_hi rows at n0, W_lo rows at N + n0.
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
    uint64_t* full = bars;                      // TMA landed
    uint64_t* empty = bars + NSTAGE;            // MMAs done with the stage
    float2* gn_sm = (float2*)(smem + NSTAGE * STAGE + 256);        // [8 consumer warps][128 columns] (sum, sum of squares)
    float* bias_s = (float*)(gn_sm + 8 * 128);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nk = (K + KC - 1) / KC;
    const int tiles_per_split = col_tiles * row_tiles;

    if (threadIdx.x == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    }
    __syncthreads();

    if (warp >= PRODUCER_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == PRODUCER_WARP && lane == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const int z = t / tiles_per_split, rem = t % tiles_per_split;
                const int m0 = (rem / col_tiles) * BM, n0 = (rem % col_tiles) * BN;
                const int kc0 = z * chunks_per_split, kc1 = min(nk, kc0 + chunks_per_split);
                for (int kc = kc0; kc < kc1; ++kc) {
                    mbar_wait(&empty[s], ph ^ 1u);
                    unsigned char* st = smem + s * STAGE;
                    mbar_arrive_expect_tx(&full[s], (uint32_t)(TILE_A + 2 * BN * 128));
                    tma_load_2d(st, &map_x, kc * KC, m0, &full[s]);
                    tma_load_2d(st + TILE_A, &map_w, kc * KC, n0, &full[s]);
                    tma_load_2d(st + TILE_A + TILE_B, &map_w, kc * KC, N + n0, &full[s]);
                    if (++s == NSTAGE) { s = 0; ph ^= 1u; }
                }
            }
        }
        return;
    }

    // ---- consumers ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
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
        // A fragment of this thread: rows g and g + 8 of the warp's 16-row slice, K columns 8kk + (lane % 4) and + 4.  In the
        // 128-byte swizzle, 16-byte chunk j of row r sits at chunk position j ^ (r % 8) = j ^ g: the 32 lanes of a load hit 32
        // different banks.
        const int g = lane >> 2, tq = lane & 3;
        const int a_off = (wg * 64 + wq * 16 + g) * 128 + tq * 4;
        // wgmma reads its register operands asynchronously: a chunk's fragments may only be overwritten once its MMAs are
        // complete, so each chunk waits for its own MMAs (wait_group 0) before the next chunk's fragments are loaded; the
        // other consumer warpgroup keeps the tensor cores busy meanwhile
        for (int kc = kc0; kc < kc1; ++kc) {
            mbar_wait(&full[s], ph);
            unsigned char* st = smem + s * STAGE;
            uint32_t f[2][KC / 8][4];           // [hi / lo][k-step][4]
#pragma unroll
            for (int kk = 0; kk < KC / 8; ++kk)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int j = 2 * kk + (e >> 1);       // 16-byte chunk of the K column
                    const float x = *reinterpret_cast<const float*>(st + a_off + (e & 1) * 8 * 128 + ((j ^ g) << 4));
                    const float hi = tf32_rn(x);        // round-to-nearest split: |lo| <= 2^-12 |x|, unbiased
                    f[0][kk][e] = __float_as_uint(hi);
                    f[1][kk][e] = __float_as_uint(x - hi);
                }
            const uint32_t sb = smem_u32(st + TILE_A);
            const uint64_t b_hi = make_desc(sb), b_lo = make_desc(sb + TILE_B);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < KC / 8; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);      // +32 bytes in 16-byte units
                const uint32_t accum = (kc == kc0 && kk == 0) ? 0u : 1u;
                wgmma_tf32_rs<BNI>(acc, f[0][kk], b_hi + adv, accum);
                wgmma_tf32_rs<BNI>(cor, f[0][kk], b_lo + adv, accum);
                wgmma_tf32_rs<BNI>(cor, f[1][kk], b_hi + adv, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();                    // this chunk's MMAs are done: its stage can be refilled
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
            if (++s == NSTAGE) { s = 0; ph ^= 1u; }
        }
        reg_fence(acc);
        reg_fence(cor);

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

// ---- per-stream scratch: split-K partials and weight images; one grow-only buffer per stream and use (like a BLAS
// workspace; freed with the process) ----------------------------------------------------------------------------------------
struct StreamWs { void* ptr; size_t bytes; };
static std::vector<std::pair<cudaStream_t, StreamWs>> g_split_ws, g_wimg_ws;
static std::mutex g_split_mu;
static float* stream_scratch(std::vector<std::pair<cudaStream_t, StreamWs>>& pool, cudaStream_t st, size_t bytes) {
    std::lock_guard<std::mutex> lk(g_split_mu);
    for (auto& e : pool)
        if (e.first == st) {
            if (e.second.bytes >= bytes) return (float*)e.second.ptr;
            // stream-ordered free: earlier kernels on this stream may still read the old buffer
            cudaFreeAsync(e.second.ptr, st);
            e.second = {nullptr, 0};
            if (cudaMallocAsync(&e.second.ptr, bytes * 2, st) != cudaSuccess) return nullptr;
            e.second.bytes = bytes * 2;
            return (float*)e.second.ptr;
        }
    StreamWs w{nullptr, 0};
    const size_t cap = bytes * 2 > (16u << 20) ? bytes * 2 : (16u << 20);
    if (cudaMallocAsync(&w.ptr, cap, st) != cudaSuccess) return nullptr;
    w.bytes = cap;
    pool.push_back({st, w});
    return (float*)w.ptr;
}

static void launch_split_tf32(const float* w, int64_t ld, int64_t n, int64_t k, float* out, cudaStream_t st) {
    const long long nk = (long long)n * k;
    long long blocks = (nk + 255) / 256;
    if (blocks > 4LL * num_sms()) blocks = 4LL * num_sms();
    ltc::split_tf32_kernel<<<(unsigned)(blocks > 0 ? blocks : 1), 256, 0, st>>>(w, ld, n, k, out);
    count_launches(1);
}

// Y = X . W^T (+ bias, row scale, ReLU, GroupNorm statistics) on the tensor cores.  w_img is the [hi | lo] tf32 image of W
// (geob200_split_tf32, 2n x k contiguous); without one, W (leading dimension ldw) is split into per-stream scratch first.
// Returns 1 when the shape/alignment is not handled by the tensor-core path (caller falls back to the fp32 kernel).
int linear_tc(const float* x, int64_t ldx, const float* w, int64_t ldw, const float* w_img, const float* bias, const float* row_scale,
              float* y, int64_t ldy, int64_t m, int64_t n, int64_t k, int relu, cudaStream_t st, const GnFuse* gn) {
    if (m < 64 || n < 32 || (n % 16) != 0 || (k % 4) != 0 || (ldx % 4) != 0) return 1;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w_img) & 15)) return 1;
    if (w_img == nullptr && ((ldw % 4) != 0 || (reinterpret_cast<uintptr_t>(w) & 15))) return 1;
    if (n > 128 && (n % 128) != 0) return 1;
    const int BN = (int)(n >= 128 ? 128 : n);
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
        part = stream_scratch(g_split_ws, st, (size_t)splits * (size_t)m * (size_t)n * sizeof(float));
        if (part == nullptr) { splits = 1; cps = nk; }
    }
    float* img = nullptr;
    if (w_img == nullptr) {
        img = stream_scratch(g_wimg_ws, st, (size_t)2 * (size_t)n * (size_t)k * sizeof(float));
        if (img == nullptr) { set_error("linear_tc: weight image scratch allocation failed"); return -1; }
        w_img = img;
    }
    CUtensorMap mx, mw;
    if (ltc::encode_map(&mx, x, m, k, ldx, ltc::BM)) return -1;
    if (ltc::encode_map(&mw, w_img, 2 * n, k, k, BN)) return -1;
    ProfRec rec{};
    const bool prof = g_prof_on;
    if (prof) {
        cudaEventCreate(&rec.a);
        cudaEventCreate(&rec.b);
        rec.m = m; rec.n = n; rec.k = k;
        cudaEventRecord(rec.a, st);
    }
    if (img != nullptr) launch_split_tf32(w, ldw, n, k, img, st);
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

// [hi | lo] tf32 image of a row-major weight (n x k, leading dimension ld): out (2n x k, contiguous) = [tf32_rn(w); w - hi]
int geob200_split_tf32(const float* w, int64_t ld, int64_t n, int64_t k, float* out, void* stream) {
    GEOB_REQUIRE(n > 0 && k > 0 && ld >= k, "split_tf32: bad shape (%lld x %lld, ld %lld)", (long long)n, (long long)k, (long long)ld);
    geob200::launch_split_tf32(w, ld, n, k, out, (cudaStream_t)stream);
    GEOB_CHECK_LAUNCH();
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
