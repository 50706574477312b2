// Hopper tensor-core (wgmma) contraction of the geometric structure embedding for C = 256 and C = 128, 3xFP16.
//
// Reference semantics: geotransformer/modules/geotransformer/geotransformer.py:57-72
//     E[p,:] = (Wd s(d_p) + bd) + max_k (Wa s(a_pk) + ba)          s(.) = C-wide interleaved sin/cos embedding
// Because the distance term does not depend on k it can be folded under the max exactly:
//     E[p,:] = max_k ( [Wa | Wd] . [s(a_pk) ; s(d_p)] ) + (ba + bd)
// so EVERY row (p,k) of the problem is one homogeneous GEMM row with K = 2C against ONE operand B = [Wa | Wd]
// (C x 2C).  A tile is 42 pairs = 126 rows (M = 128, two idle rows), N = C.
//
// Pipeline inside one persistent CTA (one per SM), 384 threads:
//   warps 0-7   consumers  : two warpgroups, tile rows [0,64) and [64,128): wgmma.m64n{C} from shared memory into a register
//                            accumulator; then the epilogue exchanges 32 columns at a time through shared memory, takes the
//                            max over the three rows of a pair, adds the bias and stores E
//   warps 8-11  generators : compute the sinusoid chunk (128 rows x 128 bytes) and store it straight into the K-major
//                            SWIZZLE_128B layout (the A operand never exists in HBM); their first thread also streams the
//                            pre-swizzled B chunk (packed once by gse_pack_b_f16_kernel) with cp.async.bulk onto the stage's mbarrier
#include <cuda_fp16.h>

#include "common.cuh"
#include "geob200.h"
#include "hopper.cuh"

namespace geob200 {
namespace tc {

using namespace hop;

constexpr int KC = 64;                 // fp16 K elements per chunk = 128 bytes = one swizzle atom row
constexpr int PAIRS = 42;              // pairs per tile
constexpr int ROWS = 128;              // tile rows (two warpgroups of M = 64)
constexpr int A_BYTES = ROWS * 128;    // 16 KB
constexpr int STAGE_LD = 33;           // epilogue exchange row stride (floats)
constexpr int NCONS_WARPS = 8;
constexpr int NGEN_WARPS = 4;
constexpr int NTHREADS = (NCONS_WARPS + NGEN_WARPS) * 32;

// sin and cos of x: Cody-Waite reduction by pi/2 to [-pi/4, pi/4], then the SFU (sin.approx / cos.approx, abs error ~4e-7 on
// that interval -- below the 2^-12 half-ulp of the fp16 hi/lo split that consumes the values).
__device__ __forceinline__ void sincos_sfu(float x, float& s, float& c) {
    if (fabsf(x) > 48000.f) { sincosf(x, &s, &c); return; }
    const float k = rintf(x * 0.636619772367581343f);
    float r = fmaf(k, -1.57079601287841796875f, x);
    r = fmaf(k, -3.1391647326017846353352069854736328125e-7f, r);
    r = fmaf(k, -5.390302529957764765e-15f, r);
    const float sp = __sinf(r), cp = __cosf(r);
    const int q = (int)k;
    const float ss = (q & 1) ? cp : sp;
    const float cc = (q & 1) ? sp : cp;
    s = (q & 2) ? -ss : ss;
    c = ((q + 1) & 2) ? -cc : cc;
}

// scale[0] = 2^-e with max|W| = m 2^e, m in [0.5,1)  ; scale[1] = 2^e
template <int CC>
__global__ void __launch_bounds__(1024) gse_absmax_kernel(const float* __restrict__ Wd, const float* __restrict__ Wa, float* __restrict__ scale) {
    __shared__ float red[32];
    float m = 0.f;
    for (int i = threadIdx.x; i < CC * CC; i += blockDim.x) m = fmaxf(m, fmaxf(fabsf(Wd[i]), fabsf(Wa[i])));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 32; ++w) m = fmaxf(m, red[w]);
        int e = 0;
        if (m > 0.f && isfinite(m)) frexpf(m, &e);
        scale[0] = ldexpf(1.0f, -e);
        scale[1] = ldexpf(1.0f, e);
    }
}

// CC = hidden dim (256: 3DMatch / ModelNet, 128: KITTI); B = [Wa | Wd] is (CC rows) x (2 CC halves), packed into per-chunk
// shared-memory images image[kc][n/8][n%8][(e/8) ^ (n%8)][e%8], hi part (fp16 of the scaled weight) and lo part (remainder).
template <int CC>
__global__ void __launch_bounds__(256) gse_pack_b_f16_kernel(const float* __restrict__ Wd, const float* __restrict__ Wa,
                                                             const float* __restrict__ bd, const float* __restrict__ ba,
                                                             const float* __restrict__ scale, __half* __restrict__ img_hi,
                                                             __half* __restrict__ img_lo, float* __restrict__ bias_sum) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < CC) bias_sum[t] = ba[t] + bd[t];
    if (t >= CC * 2 * CC) return;
    const int n = t / (2 * CC), k = t % (2 * CC);
    const float w = ((k < CC) ? Wa[n * CC + k] : Wd[n * CC + (k - CC)]) * scale[0];
    const __half hi = __float2half_rn(w);
    const int kc = k / KC, e = k % KC;
    const int dst = kc * (CC * KC) + (n >> 3) * 512 + (n & 7) * 64 + (((e >> 3) ^ (n & 7)) << 3) + (e & 7);
    img_hi[dst] = hi;
    img_lo[dst] = __float2half_rn(w - __half2float(hi));
}


// 3xFP16: x = x_hi + x_lo with x_hi = fp16(x), x_lo = fp16(x - x_hi).  fp16 carries the same 11 significant bits as tf32, so
// hi.hi + hi.lo + lo.hi has the same ~2^-22 relative accuracy as 3xTF32, but an fp16 wgmma consumes K = 16 per instruction at
// the rate a tf32 one consumes K = 8: half the tensor-pipe time, half the B bytes, half the generator stores.  The sinusoids are
// in [-1, 1] (lo <= 2^-12: fp16 subnormal spacing 6e-8 = fp32 epsilon); the weights are pre-scaled by a power of two to
// [0.5, 1) (exact), undone in the epilogue.
template <int CC>
struct Cfg {
    static constexpr int CP = CC / KC;                     // chunks per part (angle, distance)
    static constexpr int NCH = 2 * CP;                     // K chunks per tile
    static constexpr int BB = CC * 128;                    // bytes of one B chunk
    static constexpr int STAGE_BYTES = 2 * (A_BYTES + BB); // hi and lo of both operands
    static constexpr int NSTAGE = 2;
    static constexpr int SMEM = NSTAGE * STAGE_BYTES + ROWS * STAGE_LD * 4 + 1024 /*alignment slack*/ + 256 /*barriers*/;
};

// one 16-byte unit c (of 8 per 128-byte row) of the sinusoid row for argument x: frequencies f0 + 4c .. f0 + 4c + 3 (sin, cos
// interleaved), hi part and lo part
__device__ __forceinline__ void gen_unit(float x, const float* __restrict__ div_term, int f0, int c, uint4& hv, uint4& lv) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 4; ++u) sincos_sfu(__fmul_rn(x, __ldg(div_term + f0 + 4 * c + u)), v[2 * u], v[2 * u + 1]);
    __half2 hi[4], lo[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const __half h0 = __float2half_rn(v[2 * u]), h1 = __float2half_rn(v[2 * u + 1]);
        hi[u] = __halves2half2(h0, h1);
        lo[u] = __halves2half2(__float2half_rn(v[2 * u] - __half2float(h0)), __float2half_rn(v[2 * u + 1] - __half2float(h1)));
    }
    hv = make_uint4(*reinterpret_cast<uint32_t*>(&hi[0]), *reinterpret_cast<uint32_t*>(&hi[1]), *reinterpret_cast<uint32_t*>(&hi[2]),
                    *reinterpret_cast<uint32_t*>(&hi[3]));
    lv = make_uint4(*reinterpret_cast<uint32_t*>(&lo[0]), *reinterpret_cast<uint32_t*>(&lo[1]), *reinterpret_cast<uint32_t*>(&lo[2]),
                    *reinterpret_cast<uint32_t*>(&lo[3]));
}

// img_hi / img_lo: the B images of gse_pack_b_f16_kernel; scale: the weight scale of gse_absmax_kernel (scale[1] undoes it).
template <int CC>
__global__ void __launch_bounds__(NTHREADS, 1) gse_embed_kernel(const float* __restrict__ d_idx, const float* __restrict__ a_idx,
                                                                long long n_pairs, const float* __restrict__ div_term,
                                                                const __half* __restrict__ img_hi, const __half* __restrict__ img_lo,
                                                                const float* __restrict__ bias_sum, const float* __restrict__ scale,
                                                                float* __restrict__ E) {
    using CF = Cfg<CC>;
    constexpr int NSTAGE = CF::NSTAGE, R = CC / 2;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B: 1024 B alignment
    float* xstage = (float*)(smem + NSTAGE * CF::STAGE_BYTES);                                   // [128][33]
    uint64_t* bars = (uint64_t*)(xstage + ROWS * STAGE_LD);
    uint64_t* full = bars;                      // [NSTAGE] A generated + B landed
    uint64_t* empty = bars + NSTAGE;            // [NSTAGE] both consumer warpgroups are done with the stage

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long n_tiles = (n_pairs + PAIRS - 1) / PAIRS;

    if (threadIdx.x == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], NGEN_WARPS + 1); mbar_init(&empty[s], NCONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= NCONS_WARPS) {
        // ===================== generators (+ B copier) =====================
        const int gt = threadIdx.x - NCONS_WARPS * 32;
        {   // padding rows 126,127 of every A buffer: zero once (their outputs are never read)
            for (int e = gt; e < NSTAGE * 2 * 64; e += NGEN_WARPS * 32) {
                const int sidx = e / (2 * 64), rem = e % (2 * 64);
                float* base = (float*)(smem + sidx * CF::STAGE_BYTES + (rem / 64) * A_BYTES + 15 * 1024 + 6 * 128);
                base[rem % 64] = 0.f;
            }
            asm volatile("bar.sync 2, %0;" ::"n"(NGEN_WARPS * 32) : "memory");
        }
        int s = 0;
        uint32_t ph = 0;
        for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const long long p0 = tile * PAIRS;
            for (int kc = 0; kc < CF::NCH; ++kc) {
                mbar_wait(&empty[s], ph ^ 1u);
                unsigned char* st = smem + s * CF::STAGE_BYTES;
                if (gt == 0) {
                    const size_t off = (size_t)kc * CF::BB;
                    const unsigned char* hi = (const unsigned char*)img_hi + off;
                    const unsigned char* lo = (const unsigned char*)img_lo + off;
                    mbar_arrive_expect_tx(&full[s], 2 * CF::BB);
                    bulk_g2s(st + 2 * A_BYTES, hi, CF::BB, &full[s]);
                    bulk_g2s(st + 2 * A_BYTES + CF::BB, lo, CF::BB, &full[s]);
                }
                // work item = (tile row, 16-byte unit c).  Angle chunks (kc < CP) have 126 x 8 items; distance chunks have
                // 42 x 8 items whose result is stored to the three rows (k = 0,1,2) of the pair.
                const int f0 = (kc % CF::CP) * (KC / 2);
                const bool angle = kc < CF::CP;
                const int n_items = (angle ? 3 * PAIRS : PAIRS) * 8;
                for (int it = gt; it < n_items; it += NGEN_WARPS * 32) {
                    const int c = it & 7, rr = it >> 3;          // rr: tile row (angle) or pair slot (distance)
                    const int j = angle ? (rr % PAIRS) : rr;
                    const long long p = p0 + j;
                    float x = 0.f;
                    if (p < n_pairs) x = angle ? __ldg(a_idx + p * 3 + rr / PAIRS) : __ldg(d_idx + p);
                    uint4 hv, lv;
                    gen_unit(x, div_term, f0, c, hv, lv);
                    const int nrep = angle ? 1 : 3;
                    for (int rep = 0; rep < nrep; ++rep) {
                        const int r = angle ? rr : (rep * PAIRS + j);
                        const uint32_t off = (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
                        *reinterpret_cast<uint4*>(st + off) = hv;
                        *reinterpret_cast<uint4*>(st + A_BYTES + off) = lv;
                    }
                }
                fence_proxy_async();               // generic-proxy stores -> visible to the tensor core (async proxy)
                __syncwarp();
                if (lane == 0) mbar_arrive(&full[s]);
                if (++s == NSTAGE) { s = 0; ph ^= 1u; }
            }
        }
    } else {
        // ===================== consumers =====================
        const int wg = warp >> 2, wq = warp & 3;
        const float inv_scale = scale[1];
        int s = 0;
        uint32_t ph = 0;
        for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            float acc[R];
#pragma unroll
            for (int i = 0; i < R; ++i) acc[i] = 0.f;
            int prev_s = -1;
            for (int kc = 0; kc < CF::NCH; ++kc) {
                mbar_wait(&full[s], ph);
                const uint32_t st = smem_u32(smem + s * CF::STAGE_BYTES);
                const uint64_t da_hi = make_desc(st + wg * (A_BYTES / 2)), da_lo = make_desc(st + A_BYTES + wg * (A_BYTES / 2));
                const uint64_t db_hi = make_desc(st + 2 * A_BYTES), db_lo = make_desc(st + 2 * A_BYTES + CF::BB);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {       // 4 MMAs of 32 bytes of K per 128-byte chunk
                    const uint64_t adv = (uint64_t)(kk * 2);
                    wgmma_f16<CC>(acc, da_hi + adv, db_hi + adv, (kc == 0 && kk == 0) ? 0u : 1u);
                    wgmma_f16<CC>(acc, da_hi + adv, db_lo + adv, 1u);
                    wgmma_f16<CC>(acc, da_lo + adv, db_hi + adv, 1u);
                }
                wgmma_commit();
                wgmma_wait<1>();                     // the previous chunk's MMAs are done: its stage can be refilled
                if (prev_s >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev_s]); }
                prev_s = s;
                if (++s == NSTAGE) { s = 0; ph ^= 1u; }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[prev_s]);

            // epilogue, 32 columns at a time: fragment rows rl, rl + 8, columns 8j + 2(lane % 4) + {0, 1}
            const long long p0 = tile * PAIRS;
            const int rl = wg * 64 + wq * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
            for (int cc = 0; cc < CC / 32; ++cc) {
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int j = 4 * cc + jj;
                    xstage[rl * STAGE_LD + 8 * jj + c0] = acc[4 * j];
                    xstage[rl * STAGE_LD + 8 * jj + c0 + 1] = acc[4 * j + 1];
                    xstage[(rl + 8) * STAGE_LD + 8 * jj + c0] = acc[4 * j + 2];
                    xstage[(rl + 8) * STAGE_LD + 8 * jj + c0 + 1] = acc[4 * j + 3];
                }
                asm volatile("bar.sync 1, %0;" ::"n"(NCONS_WARPS * 32) : "memory");
                for (int idx = threadIdx.x; idx < PAIRS * 32; idx += NCONS_WARPS * 32) {
                    const int jp = idx >> 5, c = idx & 31;
                    const long long p = p0 + jp;
                    if (p < n_pairs) {
                        const float m = fmaxf(fmaxf(xstage[jp * STAGE_LD + c], xstage[(PAIRS + jp) * STAGE_LD + c]),
                                              xstage[(2 * PAIRS + jp) * STAGE_LD + c]);
                        E[p * CC + cc * 32 + c] = fmaf(m, inv_scale, __ldg(bias_sum + cc * 32 + c));
                    }
                }
                asm volatile("bar.sync 1, %0;" ::"n"(NCONS_WARPS * 32) : "memory");
            }
        }
    }
}

// weight scale -> packed B images -> the persistent contraction kernel, all on stream st
template <int CC>
int embed(const float* d_idx, const float* a_idx, long long n_pairs, const float* div_term, const float* Wd, const float* Wa,
          const float* bd, const float* ba, float* E, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    const size_t img_halves = (size_t)CC * 2 * CC;
    const size_t need = 2 * img_halves * sizeof(__half) + (CC + 2) * sizeof(float) + 1024;
    GEOB_REQUIRE(workspace_bytes >= need, "gse_embed_tc: workspace too small (%zu < %zu)", workspace_bytes, need);
    __half* h_hi = (__half*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    __half* h_lo = h_hi + img_halves;
    float* bsum = (float*)(h_lo + img_halves);
    float* scale = bsum + CC;
    const long long n_tiles = (n_pairs + PAIRS - 1) / PAIRS;
    const int grid = (int)(n_tiles < (long long)num_sms() ? n_tiles : (long long)num_sms());
    gse_absmax_kernel<CC><<<1, 1024, 0, st>>>(Wd, Wa, scale);
    gse_pack_b_f16_kernel<CC><<<(unsigned)((img_halves + 255) / 256), 256, 0, st>>>(Wd, Wa, bd, ba, scale, h_hi, h_lo, bsum);
    if (ensure_max_smem((const void*)gse_embed_kernel<CC>)) return -1;
    gse_embed_kernel<CC><<<grid, NTHREADS, Cfg<CC>::SMEM, st>>>(d_idx, a_idx, n_pairs, div_term, h_hi, h_lo, bsum, scale, E);
    GEOB_CHECK_LAUNCH();
    count_launches(3);
    return 0;
}

}  // namespace tc
}  // namespace geob200

using namespace geob200;

int geob200_gse_embed_tc(const float* d_idx, const float* a_idx, long long n_pairs, int C, const float* div_term,
                         const float* Wd, const float* Wa, const float* bd, const float* ba, float* E,
                         void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (C == 256) return tc::embed<256>(d_idx, a_idx, n_pairs, div_term, Wd, Wa, bd, ba, E, workspace, workspace_bytes, st);
    if (C == 128) return tc::embed<128>(d_idx, a_idx, n_pairs, div_term, Wd, Wa, bd, ba, E, workspace, workspace_bytes, st);
    return 1;
}
