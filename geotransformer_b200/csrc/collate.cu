// Stack-mode collate on the GPU: voxel-grid barycentre subsampling and batched radius neighbour search.
//
// Replaces the reference's single-threaded CPU extension `geotransformer.ext`
//   grid_subsampling  : geotransformer/extensions/cpu/grid_subsampling/grid_subsampling_cpu.cpp:3-75
//   radius_neighbors  : geotransformer/extensions/cpu/radius_neighbors/radius_neighbors_cpu.cpp:3-91
// with results that are bit-identical on continuous coordinates: same fp32 operation order (no FMA
// contraction: every product/sum goes through __fmul_rn/__fadd_rn/__fdiv_rn), same output ORDER
// (libstdc++ unordered_map iteration order emulated in parallel, see gs_order_kernel), same sentinel/padding.
//
// Everything here is HBM/L2-bound integer + fp32 work; there is no GEMM to be had.
#include <stdarg.h>
#include <string.h>

#include <mutex>
#include <set>
#include <utility>

#include "common.cuh"
#include "geob200.h"
#include "unordered_map.cuh"

namespace geob200 {

static thread_local char g_err[1024] = "";
static unsigned long long g_launches = 0;
void count_launches(int n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int ensure_max_smem(const void* kernel) {
    static std::mutex mu;
    static std::set<std::pair<const void*, int>> done;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    if (done.count({kernel, dev})) return 0;
    int optin = 0;
    cudaFuncAttributes fa{};
    cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, kernel);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
    if (e != cudaSuccess) { set_error("ensure_max_smem: %s", cudaGetErrorString(e)); return -1; }
    done.insert({kernel, dev});
    return 0;
}

// ----------------------------------------------------------------------------------------------------------
// shared small kernels
// ----------------------------------------------------------------------------------------------------------

// Per-cloud exclusive scan of an int array (one CTA per cloud, chunked with a running carry).
// out[i] = sum_{j<i, same cloud} in[j]; total[b] = sum over the cloud.  in/out may alias.
__global__ void __launch_bounds__(1024) seg_exclusive_scan_kernel(const int* __restrict__ in, int* __restrict__ out,
                                                                  const CloudSeg* __restrict__ segs,
                                                                  int* __restrict__ total) {
    __shared__ int warp_tot[32];
    __shared__ int carry_s;
    const CloudSeg sg = segs[blockIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < sg.len; base += 1024) {
        int i = base + threadIdx.x;
        int v = (i < sg.len) ? in[sg.start + i] : 0;
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_tot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int w = warp_tot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            warp_tot[lane] = w;  // inclusive
        }
        __syncthreads();
        int carry = carry_s;
        int excl = carry + (warp > 0 ? warp_tot[warp - 1] : 0) + (x - v);
        if (i < sg.len) out[sg.start + i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    if (threadIdx.x == 0 && total != nullptr) total[blockIdx.x] = carry_s;
}

// ----------------------------------------------------------------------------------------------------------
// grid subsampling
// ----------------------------------------------------------------------------------------------------------

struct GsCloud {           // per-cloud derived constants (device)
    float ox, oy, oz;      // origin corner
    unsigned long long nx, ny;
};

#define GS_EMPTY 0xFFFFFFFFFFFFFFFFull

// min/max corner, origin and grid extents: cloud.cpp:4-37, grid_subsampling_cpu.cpp:9-20
__global__ void __launch_bounds__(1024) gs_bounds_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                                         float voxel, GsCloud* __restrict__ out) {
    const CloudSeg sg = segs[blockIdx.x];
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < sg.len; i += blockDim.x) {
        const float* p = pts + 3ll * (sg.start + i);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            mn[a] = fminf(mn[a], p[a]);
            mx[a] = fmaxf(mx[a], p[a]);
        }
    }
    __shared__ float smn[3][32], smx[3][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if (lane == 0) { smn[a][warp] = mn[a]; smx[a][warp] = mx[a]; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = blockDim.x >> 5;
        for (int a = 0; a < 3; ++a)
            for (int w = 1; w < nw; ++w) {
                smn[a][0] = fminf(smn[a][0], smn[a][w]);
                smx[a][0] = fmaxf(smx[a][0], smx[a][w]);
            }
        const float inv = (float)(1.0 / (double)voxel);   // double reciprocal cast to float (cloud.h:92-94)
        GsCloud c;
        c.ox = __fmul_rn(floorf(__fmul_rn(smn[0][0], inv)), voxel);
        c.oy = __fmul_rn(floorf(__fmul_rn(smn[1][0], inv)), voxel);
        c.oz = __fmul_rn(floorf(__fmul_rn(smn[2][0], inv)), voxel);
        c.nx = (unsigned long long)(floorf(__fdiv_rn(__fsub_rn(smx[0][0], c.ox), voxel)) + 1.0f);
        c.ny = (unsigned long long)(floorf(__fdiv_rn(__fsub_rn(smx[1][0], c.oy), voxel)) + 1.0f);
        out[blockIdx.x] = c;
    }
}

// voxel key per point (grid_subsampling_cpu.cpp:32-35) + insertion into a per-cloud open-addressing table
// that records the FIRST point index of every voxel.
__global__ void gs_insert_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                 const GsCloud* __restrict__ clouds, float voxel,
                                 unsigned long long* __restrict__ tab_key, int* __restrict__ tab_first,
                                 int* __restrict__ pt_slot) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const GsCloud c = clouds[blockIdx.y];
    const float* p = pts + 3ll * (sg.start + i);
    unsigned long long ix = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(p[0], c.ox), voxel));
    unsigned long long iy = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(p[1], c.oy), voxel));
    unsigned long long iz = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(p[2], c.oz), voxel));
    unsigned long long key = ix + c.nx * iy + c.nx * c.ny * iz;
    const unsigned tsize = 2u * (unsigned)sg.len;
    const long long tbase = 2ll * sg.start;
    unsigned h = (unsigned)(mix64(key) % tsize);
    while (true) {
        unsigned long long prev = atomicCAS(&tab_key[tbase + h], GS_EMPTY, key);
        if (prev == GS_EMPTY || prev == key) break;
        h = (h + 1 == tsize) ? 0 : h + 1;
    }
    atomicMin(&tab_first[tbase + h], i);
    pt_slot[sg.start + i] = (int)h;
}

__global__ void gs_flag_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ tab_first,
                               const int* __restrict__ pt_slot, int* __restrict__ flag) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    flag[sg.start + i] = (tab_first[2ll * sg.start + pt_slot[sg.start + i]] == i) ? 1 : 0;
}

// cloud_voff[b] = sum_{b'<b} m_b' ; s_lengths (int64) for the caller
__global__ void gs_offsets_kernel(const int* __restrict__ m, int nb, int* __restrict__ voff, long long* __restrict__ s_lengths) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < nb; ++b) {
            voff[b] = acc;
            acc += m[b];
            s_lengths[b] = m[b];
        }
        voff[nb] = acc;
    }
}

// voxel ids: g = rank of the voxel's first point among first-occurrence points (per cloud).  Voxel arrays are
// stored in the cloud's POINT range [start, start+len) (m_b <= len_b), so no host sync is needed to size them.
__global__ void gs_voxel_setup_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                      const GsCloud* __restrict__ clouds, float voxel,
                                      const int* __restrict__ flag, const int* __restrict__ rank,
                                      const int* __restrict__ pt_slot, int* __restrict__ tab_rank,
                                      unsigned long long* __restrict__ vox_key) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    if (!flag[sg.start + i]) return;
    const GsCloud c = clouds[blockIdx.y];
    const float* p = pts + 3ll * (sg.start + i);
    unsigned long long ix = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(p[0], c.ox), voxel));
    unsigned long long iy = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(p[1], c.oy), voxel));
    unsigned long long iz = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(p[2], c.oz), voxel));
    const int g = rank[sg.start + i];
    tab_rank[2ll * sg.start + pt_slot[sg.start + i]] = g;
    vox_key[sg.start + g] = ix + c.nx * iy + c.nx * c.ny * iz;
}

__global__ void gs_count_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ tab_rank,
                                const int* __restrict__ pt_slot, int* __restrict__ vox_count) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const int g = tab_rank[2ll * sg.start + pt_slot[sg.start + i]];
    atomicAdd(&vox_count[sg.start + g], 1);
}

__global__ void gs_scatter_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ tab_rank,
                                  const int* __restrict__ pt_slot, const int* __restrict__ vox_off,
                                  int* __restrict__ vox_cursor, int* __restrict__ vox_pts) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const int g = tab_rank[2ll * sg.start + pt_slot[sg.start + i]];
    const int pos = atomicAdd(&vox_cursor[sg.start + g], 1);
    vox_pts[sg.start + vox_off[sg.start + g] + pos] = i;
}

// Barycentre of every voxel with the reference's accumulation order: fp32 sum in INPUT order
// (grid_subsampling_cpu.h:17-20), times float(1.0/count) (grid_subsampling_cpu.cpp:46).
// The voxel's point list was filled by atomics in arbitrary order; points are consumed by repeatedly taking
// the smallest index larger than the last one (lists are short: a few points per voxel).
__global__ void gs_reduce_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                 const int* __restrict__ m_per_cloud, const int* __restrict__ vox_off,
                                 const int* __restrict__ vox_count, const int* __restrict__ vox_pts,
                                 float* __restrict__ vox_bary) {
    const CloudSeg sg = segs[blockIdx.y];
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= m_per_cloud[blockIdx.y]) return;
    const int c = vox_count[sg.start + g];
    const int* lst = vox_pts + sg.start + vox_off[sg.start + g];
    float sx = 0.f, sy = 0.f, sz = 0.f;
    int last = -1;
    for (int k = 0; k < c; ++k) {
        int best = 0x7fffffff;
        for (int j = 0; j < c; ++j) {
            int v = lst[j];
            if (v > last && v < best) best = v;
        }
        const float* p = pts + 3ll * (sg.start + best);
        sx = __fadd_rn(sx, p[0]);
        sy = __fadd_rn(sy, p[1]);
        sz = __fadd_rn(sz, p[2]);
        last = best;
    }
    const float w = (float)(1.0 / (double)c);
    float* o = vox_bary + 3ll * (sg.start + g);
    o[0] = __fmul_rn(sx, w);
    o[1] = __fmul_rn(sy, w);
    o[2] = __fmul_rn(sz, w);
}

// Output order of grid subsampling = iteration order of std::unordered_map<size_t, ...> after inserting the voxel keys in
// first-occurrence order (grid_subsampling_cpu.cpp:26-47); std::hash<size_t> is the identity, so a key is its own bucket hash.
// One CTA per cloud: the order, then the gather of the fp32 barycentres.
__global__ void __launch_bounds__(1024) gs_order_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ m_per_cloud,
                                                        const int* __restrict__ cloud_voff,
                                                        const unsigned long long* __restrict__ vox_key,
                                                        const float* __restrict__ vox_bary,
                                                        int* __restrict__ cur_g, int* __restrict__ nxt_g,
                                                        int* __restrict__ A_g, int* __restrict__ lnk_g,
                                                        int* __restrict__ bucket_scratch,   // 3 ints per bucket
                                                        float* __restrict__ s_points) {
    const CloudSeg sg = segs[blockIdx.x];
    const int m = m_per_cloud[blockIdx.x];
    // bucket arrays: capacity 3*len+64 per cloud (nb <= 2.2*m+13)
    int* act = bucket_scratch + (3ll * sg.start + 64ll * blockIdx.x) * 3;
    const long long bcap = 3ll * sg.len + 64;
    const int* order = unordered_map_order(m, vox_key + sg.start, cur_g + sg.start, nxt_g + sg.start, A_g + sg.start,
                                           lnk_g + sg.start, act, act + bcap, act + 2 * bcap);
    // m == 0 cannot happen for a non-empty cloud; order[] lists voxel ids head -> tail.
    float* out = s_points + 3ll * cloud_voff[blockIdx.x];
    for (int q = threadIdx.x; q < m; q += blockDim.x) {
        const float* bsrc = vox_bary + 3ll * (sg.start + order[q]);
        out[3 * q + 0] = bsrc[0];
        out[3 * q + 1] = bsrc[1];
        out[3 * q + 2] = bsrc[2];
    }
}

static int upload_segs(const int64_t* lengths_h, int64_t batch, CloudSeg* d_segs, int64_t* total, int* max_len,
                       cudaStream_t st) {
    CloudSeg tmp[64];
    CloudSeg* h = tmp;
    CloudSeg* heap = nullptr;
    if (batch > 64) { heap = (CloudSeg*)malloc(sizeof(CloudSeg) * batch); h = heap; }
    int64_t acc = 0;
    int mx = 0;
    for (int64_t b = 0; b < batch; ++b) {
        h[b].start = (int)acc;
        h[b].len = (int)lengths_h[b];
        acc += lengths_h[b];
        if ((int)lengths_h[b] > mx) mx = (int)lengths_h[b];
    }
    cudaError_t e = cudaMemcpyAsync(d_segs, h, sizeof(CloudSeg) * batch, cudaMemcpyHostToDevice, st);
    if (heap) { cudaStreamSynchronize(st); free(heap); }
    *total = acc;
    *max_len = mx;
    if (e != cudaSuccess) { set_error("upload_segs: %s", cudaGetErrorString(e)); return -1; }
    return 0;
}

// ----------------------------------------------------------------------------------------------------------
// radius search
// ----------------------------------------------------------------------------------------------------------

struct RsCloud {
    float ox, oy, oz;   // min corner of the SUPPORT cloud
    float cell;         // cell edge (>= radius * 1.001)
    int cx, cy, cz;     // grid extents
    int cell_base;      // offset of this cloud's cells in the global cell arrays
};

// support bounding box -> uniform grid with cell >= 1.001 r, shrunk to the per-cloud cell budget
__global__ void __launch_bounds__(1024) rs_bounds_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                                         float radius, RsCloud* __restrict__ out, CloudSeg* __restrict__ cell_segs,
                                                         int* __restrict__ max_count) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *max_count = 0;
    const CloudSeg sg = segs[blockIdx.x];
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < sg.len; i += blockDim.x) {
        const float* p = pts + 3ll * (sg.start + i);
#pragma unroll
        for (int a = 0; a < 3; ++a) { mn[a] = fminf(mn[a], p[a]); mx[a] = fmaxf(mx[a], p[a]); }
    }
    __shared__ float smn[3][32], smx[3][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if (lane == 0) { smn[a][warp] = mn[a]; smx[a][warp] = mx[a]; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = blockDim.x >> 5;
        for (int a = 0; a < 3; ++a)
            for (int w = 1; w < nw; ++w) { smn[a][0] = fminf(smn[a][0], smn[a][w]); smx[a][0] = fmaxf(smx[a][0], smx[a][w]); }
        RsCloud c;
        c.ox = smn[0][0]; c.oy = smn[1][0]; c.oz = smn[2][0];
        const long long budget = 2ll * sg.len + 1024;
        float cell = radius * 1.001f;
        long long cx, cy, cz;
        while (true) {
            cx = (long long)floorf((smx[0][0] - c.ox) / cell) + 1;
            cy = (long long)floorf((smx[1][0] - c.oy) / cell) + 1;
            cz = (long long)floorf((smx[2][0] - c.oz) / cell) + 1;
            if (cx <= 1024 && cy <= 1024 && cz <= 1024 && cx * cy * cz <= budget) break;
            cell *= 1.25f;
        }
        c.cell = cell; c.cx = (int)cx; c.cy = (int)cy; c.cz = (int)cz;
        c.cell_base = 2 * sg.start + 1025 * blockIdx.x;   // budget+1 cells (one extra for the end offset)
        out[blockIdx.x] = c;
        cell_segs[blockIdx.x].start = c.cell_base;
        cell_segs[blockIdx.x].len = c.cx * c.cy * c.cz + 1;   // +1: the trailing entry receives the cloud total
    }
}

__device__ __forceinline__ int rs_cell_of(const RsCloud& c, float x, float y, float z) {
    int ix = (int)floorf((x - c.ox) / c.cell), iy = (int)floorf((y - c.oy) / c.cell), iz = (int)floorf((z - c.oz) / c.cell);
    ix = min(max(ix, 0), c.cx - 1); iy = min(max(iy, 0), c.cy - 1); iz = min(max(iz, 0), c.cz - 1);
    return (iz * c.cy + iy) * c.cx + ix;
}

__global__ void rs_count_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                const RsCloud* __restrict__ clouds, int* __restrict__ cell_cnt, int* __restrict__ pt_cell) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const RsCloud c = clouds[blockIdx.y];
    const float* p = pts + 3ll * (sg.start + i);
    const int cell = rs_cell_of(c, p[0], p[1], p[2]);
    pt_cell[sg.start + i] = cell;
    atomicAdd(&cell_cnt[c.cell_base + cell], 1);
}

__global__ void rs_scatter_kernel(const float* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                  const RsCloud* __restrict__ clouds, const int* __restrict__ cell_start,
                                  int* __restrict__ cell_cursor, const int* __restrict__ pt_cell,
                                  float4* __restrict__ sorted) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const RsCloud c = clouds[blockIdx.y];
    const int cell = pt_cell[sg.start + i];
    const int pos = atomicAdd(&cell_cursor[c.cell_base + cell], 1);
    const float* p = pts + 3ll * (sg.start + i);
    sorted[sg.start + cell_start[c.cell_base + cell] + pos] = make_float4(p[0], p[1], p[2], __int_as_float(i));
}

struct RsSegs {  // cell scan segments: one per cloud over its cell range
    int start, len;
};
__global__ void rs_cellsegs_kernel(const RsCloud* __restrict__ clouds, int nb, CloudSeg* __restrict__ cell_segs) {
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const RsCloud c = clouds[b];
    cell_segs[b].start = c.cell_base;
    cell_segs[b].len = c.cx * c.cy * c.cz + 1;   // +1: the trailing entry receives the cloud total
}

// One warp per query.  Candidates from the 27 surrounding cells (9 x-contiguous runs) are tested with the
// reference metric  d2 = ((dx*dx) + dy*dy) + dz*dz  (nanoflann.hpp:432-440), strict d2 < r*r
// (nanoflann.hpp:249-253), collected as (d2 bits << 32 | index) keys in shared memory, bitonic-sorted
// (ascending distance, ties by index) and the first `width` written with the cloud offset added; missing
// entries get the sentinel n_support_total (radius_neighbors_cpu.cpp:78-88).
// Warp-level bitonic sort of 32 * KPL 64-bit keys held in registers, striped layout: element e = r * 32 + lane lives in
// register r of lane `lane`.  Partners less than 32 apart are exchanged with shuffles, the others are register pairs of the same
// lane: no shared-memory round trips and no __syncwarp per step (a shared-memory sort spends most of the query in them).
template <int KPL>
__device__ __forceinline__ void warp_bitonic_sort(unsigned long long (&key)[KPL], int lane) {
#pragma unroll
    for (int k = 2; k <= 32 * KPL; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            if (j >= 32) {
                const int rj = j >> 5;
#pragma unroll
                for (int r = 0; r < KPL; ++r) {
                    if ((r & rj) == 0) {
                        const bool up = (((r * 32 + lane) & k) == 0);
                        const unsigned long long a = key[r], b = key[r | rj];
                        const bool swap = (a > b) == up;
                        key[r] = swap ? b : a;
                        key[r | rj] = swap ? a : b;
                    }
                }
            } else {
#pragma unroll
                for (int r = 0; r < KPL; ++r) {
                    const unsigned long long a = key[r];
                    const unsigned long long b = __shfl_xor_sync(0xffffffffu, a, j);
                    const bool up = (((r * 32 + lane) & k) == 0);
                    const bool lower = (lane & j) == 0;
                    const bool take_min = (up == lower);
                    key[r] = take_min ? (a < b ? a : b) : (a > b ? a : b);
                }
            }
        }
    }
}

template <int KPL>
__device__ __forceinline__ void rs_sort_and_store(const unsigned long long* buf, int count, int lane, long long* orow, int width,
                                                  long long start, long long sentinel) {
    unsigned long long key[KPL];
#pragma unroll
    for (int r = 0; r < KPL; ++r) key[r] = (r * 32 + lane < count) ? buf[r * 32 + lane] : 0xFFFFFFFFFFFFFFFFull;
    warp_bitonic_sort<KPL>(key, lane);
#pragma unroll
    for (int r = 0; r < KPL; ++r) {
        const int e = r * 32 + lane;
        if (e < width) orow[e] = (e < count) ? (long long)(unsigned)(key[r] & 0xFFFFFFFFull) + start : sentinel;
    }
    for (int e = 32 * KPL + lane; e < width; e += 32) orow[e] = sentinel;       // table wider than the sorted block
}

template <int CAP>
__device__ __forceinline__ void rs_query_body(unsigned long long* buf, int lane, int b, int qi,
                                              const float* __restrict__ q_pts, const CloudSeg* __restrict__ q_segs,
                                              const CloudSeg* __restrict__ s_segs, const RsCloud* __restrict__ clouds,
                                              const int* __restrict__ cell_start, const float4* __restrict__ sorted,
                                              float radius, int width, long long sentinel, long long* __restrict__ out,
                                              int* __restrict__ counts, int* __restrict__ max_count,
                                              int* __restrict__ overflow_list, int* __restrict__ overflow_n) {
    const CloudSeg qs = q_segs[b];
    const CloudSeg ss = s_segs[b];
    const RsCloud c = clouds[b];
    const long long row = (long long)qs.start + qi;
    const float qx = q_pts[3 * row], qy = q_pts[3 * row + 1], qz = q_pts[3 * row + 2];
    const float r2 = __fmul_rn(radius, radius);
    const float lim = 2.0e6f;
    const int ix = (int)fminf(fmaxf(floorf((qx - c.ox) / c.cell), -lim), lim);
    const int iy = (int)fminf(fmaxf(floorf((qy - c.oy) / c.cell), -lim), lim);
    const int iz = (int)fminf(fmaxf(floorf((qz - c.oz) / c.cell), -lim), lim);
    int count = 0;
    const int x0 = max(ix - 1, 0), x1 = min(ix + 1, c.cx - 1);
    if (x0 <= x1) {
        for (int dz = -1; dz <= 1; ++dz) {
            const int z = iz + dz;
            if (z < 0 || z >= c.cz) continue;
            for (int dy = -1; dy <= 1; ++dy) {
                const int y = iy + dy;
                if (y < 0 || y >= c.cy) continue;
                const int rowcell = c.cell_base + (z * c.cy + y) * c.cx;
                const int beg = cell_start[rowcell + x0], end = cell_start[rowcell + x1 + 1];
                const int end_pad = beg + ((end - beg + 31) / 32) * 32;
                for (int k = beg + lane; k < end_pad; k += 32) {
                    bool hit = false;
                    unsigned long long kv = 0;
                    if (k < end) {
                        const float4 s = sorted[ss.start + k];
                        const float ex = __fsub_rn(qx, s.x), ey = __fsub_rn(qy, s.y), ez = __fsub_rn(qz, s.z);
                        float d = __fmul_rn(ex, ex);
                        d = __fadd_rn(d, __fmul_rn(ey, ey));
                        d = __fadd_rn(d, __fmul_rn(ez, ez));
                        hit = d < r2;
                        kv = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(s.w);
                    }
                    const unsigned msk = __ballot_sync(0xffffffffu, hit);
                    if (hit) {
                        const int pos = count + __popc(msk & ((1u << lane) - 1u));
                        if (pos < CAP) buf[pos] = kv;
                    }
                    count += __popc(msk);
                }
            }
        }
    }
    if (count > CAP) {
        // too many neighbours for this buffer: hand the query to the large-capacity pass (or flag failure)
        if (lane == 0) {
            if (overflow_list != nullptr) overflow_list[atomicAdd(overflow_n, 1)] = (int)row;
            else atomicExch(max_count, -1 << 30);   // poisons max_count: callers treat a negative value as an error
        }
        return;
    }
    if (lane == 0) {
        if (counts != nullptr) counts[row] = count;
        atomicMax(max_count, count);
    }
    if (out == nullptr || width <= 0) return;
    // ascending by (d2 bits, index): register-resident warp bitonic sort of the next power of two >= count keys
    __syncwarp();
    long long* orow = out + row * (long long)width;
    if (count <= 32) rs_sort_and_store<1>(buf, count, lane, orow, width, ss.start, sentinel);
    else if (count <= 64) rs_sort_and_store<2>(buf, count, lane, orow, width, ss.start, sentinel);
    else if (count <= 128) rs_sort_and_store<4>(buf, count, lane, orow, width, ss.start, sentinel);
    else if (count <= 256) rs_sort_and_store<8>(buf, count, lane, orow, width, ss.start, sentinel);
    else {
        // large-capacity pass (rs_redo_kernel): shared-memory bitonic sort
        int n2 = 1;
        while (n2 < count) n2 <<= 1;
        for (int k = count + lane; k < n2; k += 32) buf[k] = 0xFFFFFFFFFFFFFFFFull;
        __syncwarp();
        for (int k = 2; k <= n2; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int t = lane; t < n2; t += 32) {
                    const int p = t ^ j;
                    if (p > t) {
                        const unsigned long long a = buf[t], bb = buf[p];
                        const bool up = ((t & k) == 0);
                        if ((a > bb) == up) { buf[t] = bb; buf[p] = a; }
                    }
                }
                __syncwarp();
            }
        }
        for (int k = lane; k < width; k += 32)
            orow[k] = (k < count) ? (long long)(unsigned)(buf[k] & 0xFFFFFFFFull) + ss.start : sentinel;
    }
}

template <int CAP>
__global__ void rs_query_kernel(const float* __restrict__ q_pts, const CloudSeg* __restrict__ q_segs,
                                const CloudSeg* __restrict__ s_segs, const RsCloud* __restrict__ clouds,
                                const int* __restrict__ cell_start, const float4* __restrict__ sorted, float radius,
                                int width, long long sentinel, long long* __restrict__ out, int* __restrict__ counts,
                                int* __restrict__ max_count, int* __restrict__ overflow_list, int* __restrict__ overflow_n) {
    extern __shared__ unsigned long long smem_keys[];
    const int warps_per_block = blockDim.x >> 5;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    const int qi = blockIdx.x * warps_per_block + warp;
    if (qi >= q_segs[b].len) return;
    rs_query_body<CAP>(smem_keys + (size_t)warp * CAP, lane, b, qi, q_pts, q_segs, s_segs, clouds, cell_start, sorted,
                       radius, width, sentinel, out, counts, max_count, overflow_list, overflow_n);
}

// Large-capacity second pass over the (normally empty) overflow list; one warp per CTA, grid-stride.
template <int CAP>
__global__ void rs_redo_kernel(const float* __restrict__ q_pts, const CloudSeg* __restrict__ q_segs,
                               const CloudSeg* __restrict__ s_segs, const RsCloud* __restrict__ clouds,
                               const int* __restrict__ cell_start, const float4* __restrict__ sorted, float radius,
                               int width, long long sentinel, long long* __restrict__ out, int* __restrict__ counts,
                               int* __restrict__ max_count, const int* __restrict__ redo_list,
                               const int* __restrict__ redo_n, int nbatch) {
    extern __shared__ unsigned long long smem_keys[];
    const int n = *redo_n;
    for (int w = blockIdx.x; w < n; w += gridDim.x) {
        const int row = redo_list[w];
        int b = 0;
        while (b + 1 < nbatch && row >= q_segs[b + 1].start) ++b;
        rs_query_body<CAP>(smem_keys, threadIdx.x, b, row - q_segs[b].start, q_pts, q_segs, s_segs, clouds, cell_start,
                           sorted, radius, width, sentinel, out, counts, max_count, nullptr, nullptr);
        __syncwarp();
    }
}

// calibrate_neighbors_stack_mode (utils/data.py:190-217): histogram of the number of valid entries per neighbour-table row
// (np.sum(neighbors < n_support, axis=1) -> np.bincount(...)[:hist_n]).  One thread per row, counts beyond hist_n dropped.
__global__ void __launch_bounds__(256) neighbor_histogram_kernel(const long long* __restrict__ nbr, long long rows, int width,
                                                                 long long n_support, int hist_n, int* __restrict__ hist) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    int c = 0;
    for (int j = 0; j < width; ++j) c += nbr[r * width + j] < n_support ? 1 : 0;
    if (c < hist_n) atomicAdd(&hist[c], 1);
}

// the batched calibration's stage tables: pointers, widths, row counts and each cloud's first row per stage
struct HistStages {
    const long long* nbr[GEOB200_MAX_STAGES];
    long long rows[GEOB200_MAX_STAGES];
    int width[GEOB200_MAX_STAGES];
    int cloud_start[GEOB200_MAX_STAGES][2 * GEOB200_HIST_MAX_PAIRS + 1];
};

// one thread per row of stage blockIdx.y: the row's valid-entry count goes to the histogram of its pair (cloud c is pair c mod B)
__global__ void __launch_bounds__(256) neighbor_histogram_batched_kernel(HistStages st, int num_stages, int batch, int hist_n,
                                                                         int* __restrict__ hists) {
    const int s = blockIdx.y;
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= st.rows[s]) return;
    const int w = st.width[s];
    const long long* row = st.nbr[s] + r * w;
    int c = 0;
    for (int j = 0; j < w; ++j) c += row[j] < st.rows[s] ? 1 : 0;
    if (c >= hist_n) return;
    int cloud = 0;
    while (cloud + 1 < 2 * batch && r >= st.cloud_start[s][cloud + 1]) ++cloud;
    atomicAdd(&hists[((size_t)(cloud % batch) * num_stages + s) * hist_n + c], 1);
}

// the reference's early exit over the batch's pairs in order, continuing the running totals of earlier calls
__global__ void __launch_bounds__(256) neighbor_histogram_stop_kernel(const int* __restrict__ hists, int num_stages, int batch,
                                                                      int hist_n, long long threshold, int* __restrict__ totals,
                                                                      int* __restrict__ stop) {
    __shared__ long long row_sum[GEOB200_HIST_MAX_PAIRS * GEOB200_MAX_STAGES];
    __shared__ long long base[GEOB200_MAX_STAGES];
    __shared__ int last;
    const int t = threadIdx.x;
    for (int i = t; i < batch * num_stages; i += blockDim.x) {
        long long v = 0;
        for (int h = 0; h < hist_n; ++h) v += hists[(size_t)i * hist_n + h];
        row_sum[i] = v;
    }
    for (int s = t; s < num_stages; s += blockDim.x) {
        long long v = 0;
        for (int h = 0; h < hist_n; ++h) v += totals[(size_t)s * hist_n + h];
        base[s] = v;
    }
    __syncthreads();
    if (t == 0) {
        int found = -1;
        for (int p = 0; p < batch && found < 0; ++p) {
            bool all = true;
            for (int s = 0; s < num_stages; ++s) {
                base[s] += row_sum[p * num_stages + s];
                all = all && base[s] > threshold;
            }
            if (all) found = p;
        }
        *stop = found;
        last = found >= 0 ? found : batch - 1;
    }
    __syncthreads();
    for (int i = t; i < num_stages * hist_n; i += blockDim.x) {
        int v = totals[i];
        for (int p = 0; p <= last; ++p) v += hists[(size_t)p * num_stages * hist_n + i];
        totals[i] = v;
    }
}

}  // namespace geob200

using namespace geob200;

extern "C" {

const char* geob200_last_error(void) { return g_err; }
uint64_t geob200_launch_count(void) { return g_launches; }

size_t geob200_grid_subsample_workspace_bytes(int64_t n_points, int64_t batch) {
    size_t n = (size_t)n_points, b = (size_t)batch;
    size_t bytes = 0;
    bytes += align_up(sizeof(CloudSeg) * b, 256) + align_up(sizeof(GsCloud) * b, 256);
    bytes += align_up(8 * 2 * n, 256) + align_up(4 * 2 * n, 256) * 2;      // tab_key, tab_first, tab_rank
    bytes += align_up(4 * n, 256) * 11;                                     // pt_slot, flag, rank, count, off, cursor, pts, cur, nxt, A, lnk
    bytes += align_up(8 * n, 256);                                          // vox_key
    bytes += align_up(12 * n, 256);                                         // vox_bary
    bytes += align_up(4 * 3 * (3 * n + 64 * b), 256);                       // bucket scratch
    bytes += align_up(4 * (b + 1), 256) * 2;                                // m_per_cloud, voff
    return bytes + 4096;
}

int geob200_grid_subsample(const float* points, int64_t n_points, const int64_t* lengths_h, int64_t batch, float voxel,
                           float* s_points, int64_t* s_lengths, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(batch > 0 && n_points > 0, "grid_subsample: empty input (n=%lld, batch=%lld)", (long long)n_points, (long long)batch);
    GEOB_REQUIRE(voxel > 0.f, "grid_subsample: voxel size must be positive");
    GEOB_REQUIRE(n_points < (1ll << 30), "grid_subsample: too many points");
    for (int64_t b = 0; b < batch; ++b)
        GEOB_REQUIRE(lengths_h[b] > 0, "grid_subsample: cloud %lld is empty (the reference reads points[0])", (long long)b);
    GEOB_REQUIRE(workspace_bytes >= geob200_grid_subsample_workspace_bytes(n_points, batch), "grid_subsample: workspace too small");
    Arena ar(workspace, workspace_bytes);
    const size_t n = (size_t)n_points;
    CloudSeg* segs = ar.take<CloudSeg>(batch);
    GsCloud* clouds = ar.take<GsCloud>(batch);
    unsigned long long* tab_key = ar.take<unsigned long long>(2 * n);
    int* tab_first = ar.take<int>(2 * n);
    int* tab_rank = ar.take<int>(2 * n);
    int* pt_slot = ar.take<int>(n);
    int* flag = ar.take<int>(n);
    int* rank = ar.take<int>(n);
    int* vox_count = ar.take<int>(2 * n);      // [vox_count | vox_cursor], zeroed together
    int* vox_cursor = vox_count + n;
    int* vox_off = ar.take<int>(n);
    int* vox_pts = ar.take<int>(n);
    int* cur = ar.take<int>(n);
    int* nxt = ar.take<int>(n);
    int* A = ar.take<int>(n);
    int* lnk = ar.take<int>(n);
    unsigned long long* vox_key = ar.take<unsigned long long>(n);
    float* vox_bary = ar.take<float>(3 * n);
    int* bucket_scratch = ar.take<int>(3 * (3 * n + 64 * (size_t)batch));
    int* m_per_cloud = ar.take<int>(batch + 1);
    int* voff = ar.take<int>(batch + 1);
    GEOB_REQUIRE(ar.ok(), "grid_subsample: workspace accounting error");

    int64_t total = 0;
    int max_len = 0;
    if (upload_segs(lengths_h, batch, segs, &total, &max_len, st)) return -1;
    GEOB_REQUIRE(total == n_points, "grid_subsample: sum(lengths)=%lld != n_points=%lld", (long long)total, (long long)n_points);

    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_key, 0xFF, 8 * 2 * n, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_first, 0x7F, 4 * 2 * n, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(vox_count, 0, 4 * 2 * n, st));

    const dim3 pgrid((max_len + 255) / 256, (unsigned)batch);
    gs_bounds_kernel<<<(unsigned)batch, 1024, 0, st>>>(points, segs, voxel, clouds);
    gs_insert_kernel<<<pgrid, 256, 0, st>>>(points, segs, clouds, voxel, tab_key, tab_first, pt_slot);
    gs_flag_kernel<<<pgrid, 256, 0, st>>>(segs, tab_first, pt_slot, flag);
    seg_exclusive_scan_kernel<<<(unsigned)batch, 1024, 0, st>>>(flag, rank, segs, m_per_cloud);
    gs_offsets_kernel<<<1, 32, 0, st>>>(m_per_cloud, (int)batch, voff, (long long*)s_lengths);
    gs_voxel_setup_kernel<<<pgrid, 256, 0, st>>>(points, segs, clouds, voxel, flag, rank, pt_slot, tab_rank, vox_key);
    gs_count_kernel<<<pgrid, 256, 0, st>>>(segs, tab_rank, pt_slot, vox_count);
    seg_exclusive_scan_kernel<<<(unsigned)batch, 1024, 0, st>>>(vox_count, vox_off, segs, nullptr);
    gs_scatter_kernel<<<pgrid, 256, 0, st>>>(segs, tab_rank, pt_slot, vox_off, vox_cursor, vox_pts);
    gs_reduce_kernel<<<pgrid, 256, 0, st>>>(points, segs, m_per_cloud, vox_off, vox_count, vox_pts, vox_bary);
    gs_order_kernel<<<(unsigned)batch, 1024, 0, st>>>(segs, m_per_cloud, voff, vox_key, vox_bary, cur, nxt, A, lnk,
                                                     bucket_scratch, s_points);
    GEOB_CHECK_LAUNCH();
    count_launches(11);
    return 0;
}

size_t geob200_radius_search_workspace_bytes(int64_t n_query, int64_t n_support, int64_t batch) {
    size_t ns = (size_t)n_support, nq = (size_t)n_query, b = (size_t)batch;
    size_t cells = 2 * ns + 1025 * b + 64;
    size_t bytes = 0;
    bytes += align_up(sizeof(CloudSeg) * b, 256) * 3 + align_up(sizeof(RsCloud) * b, 256);
    bytes += align_up(4 * cells, 256) * 3 + 1024;     // cnt, start, cursor (+ counters)
    bytes += align_up(4 * ns, 256);            // pt_cell
    bytes += align_up(16 * ns, 256);           // sorted float4
    bytes += align_up(4 * nq, 256);            // overflow list
    bytes += 1024;
    return bytes + 4096;
}

int geob200_radius_search(const float* q_points, int64_t n_query, const float* s_points, int64_t n_support,
                          const int64_t* q_lengths_h, const int64_t* s_lengths_h, int64_t batch, float radius,
                          int64_t width, int64_t* out, int32_t* counts, int32_t* max_count, void* workspace,
                          size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(batch > 0 && n_query > 0 && n_support > 0, "radius_search: empty input");
    GEOB_REQUIRE(radius > 0.f, "radius_search: radius must be positive");
    GEOB_REQUIRE(max_count != nullptr, "radius_search: max_count output is required");
    GEOB_REQUIRE(n_query < (1ll << 30) && n_support < (1ll << 30), "radius_search: too many points");
    GEOB_REQUIRE(workspace_bytes >= geob200_radius_search_workspace_bytes(n_query, n_support, batch), "radius_search: workspace too small");
    for (int64_t b = 0; b < batch; ++b)
        GEOB_REQUIRE(q_lengths_h[b] >= 0 && s_lengths_h[b] > 0, "radius_search: cloud %lld has no support points", (long long)b);
    Arena ar(workspace, workspace_bytes);
    const size_t ns = (size_t)n_support;
    const size_t cells = 2 * ns + 1025 * (size_t)batch + 64;
    CloudSeg* q_segs = ar.take<CloudSeg>(batch);
    CloudSeg* s_segs = ar.take<CloudSeg>(batch);
    CloudSeg* cell_segs = ar.take<CloudSeg>(batch);
    RsCloud* clouds = ar.take<RsCloud>(batch);
    // one zero-filled block: [cell_cnt | cell_cursor | overflow counters]
    int* zero_block = ar.take<int>(2 * cells + 64);
    int* cell_cnt = zero_block;
    int* cell_cursor = zero_block + cells;
    int* overflow_n = zero_block + 2 * cells;
    int* cell_start = ar.take<int>(cells);
    int* pt_cell = ar.take<int>(ns);
    float4* sorted = ar.take<float4>(ns);
    int* overflow_list = ar.take<int>((size_t)n_query);
    GEOB_REQUIRE(ar.ok(), "radius_search: workspace accounting error");

    int64_t tq = 0, ts = 0;
    int max_q = 0, max_s = 0;
    if (upload_segs(q_lengths_h, batch, q_segs, &tq, &max_q, st)) return -1;
    if (upload_segs(s_lengths_h, batch, s_segs, &ts, &max_s, st)) return -1;
    GEOB_REQUIRE(tq == n_query && ts == n_support, "radius_search: lengths do not sum to the row counts");

    GEOB_CHECK_CUDA(cudaMemsetAsync(zero_block, 0, 4 * (2 * cells + 64), st));

    const dim3 sgrid((max_s + 255) / 256, (unsigned)batch);
    rs_bounds_kernel<<<(unsigned)batch, 1024, 0, st>>>(s_points, s_segs, radius, clouds, cell_segs, max_count);
    rs_count_kernel<<<sgrid, 256, 0, st>>>(s_points, s_segs, clouds, cell_cnt, pt_cell);
    seg_exclusive_scan_kernel<<<(unsigned)batch, 1024, 0, st>>>(cell_cnt, cell_start, cell_segs, nullptr);
    rs_scatter_kernel<<<sgrid, 256, 0, st>>>(s_points, s_segs, clouds, cell_start, cell_cursor, pt_cell, sorted);
    if (max_q > 0) {
        constexpr int CAP = 256, WARPS = 4;
        const dim3 qgrid((max_q + WARPS - 1) / WARPS, (unsigned)batch);
        rs_query_kernel<CAP><<<qgrid, WARPS * 32, WARPS * CAP * 8, st>>>(
            q_points, q_segs, s_segs, clouds, cell_start, sorted, radius, (int)width, (long long)n_support,
            (long long*)out, counts, max_count, overflow_list, overflow_n);
        // queries with more than CAP neighbours (none at the reference's densities) are redone with a
        // 16384-entry buffer; the launch is a no-op when the overflow list is empty, so no host sync is needed.
        constexpr int CAP2 = 16384;
        if (ensure_max_smem((const void*)rs_redo_kernel<CAP2>)) return -1;
        rs_redo_kernel<CAP2><<<num_sms(), 32, CAP2 * 8, st>>>(
            q_points, q_segs, s_segs, clouds, cell_start, sorted, radius, (int)width, (long long)n_support,
            (long long*)out, counts, max_count, overflow_list, overflow_n, (int)batch);
        count_launches(2);
    }
    GEOB_CHECK_LAUNCH();
    count_launches(4);
    return 0;
}

int geob200_neighbor_histogram(const int64_t* neighbors, int64_t n_rows, int64_t width, int64_t n_support, int64_t hist_n,
                               int32_t* hist, void* stream) {
    GEOB_REQUIRE(n_rows > 0 && width > 0 && hist_n > 0, "neighbor_histogram: empty input");
    neighbor_histogram_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (const long long*)neighbors, (long long)n_rows, (int)width, (long long)n_support, (int)hist_n, hist);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

int geob200_neighbor_histogram_batched(const int64_t* const* neighbors, const int64_t* widths, const int64_t* cloud_rows,
                                       int64_t num_stages, int64_t batch, int64_t hist_n, int64_t sample_threshold, int32_t* hists,
                                       int32_t* totals, int32_t* stop, void* stream) {
    GEOB_REQUIRE(num_stages >= 1 && num_stages <= GEOB200_MAX_STAGES, "neighbor_histogram_batched: num_stages must be in 1..%d",
                 GEOB200_MAX_STAGES);
    GEOB_REQUIRE(batch >= 1 && batch <= GEOB200_HIST_MAX_PAIRS, "neighbor_histogram_batched: batch must be in 1..%d",
                 GEOB200_HIST_MAX_PAIRS);
    GEOB_REQUIRE(hist_n >= 1 && hist_n <= (1 << 20), "neighbor_histogram_batched: hist_n must be in 1..2^20");
    GEOB_REQUIRE(neighbors != nullptr && widths != nullptr && cloud_rows != nullptr && hists != nullptr && totals != nullptr &&
                 stop != nullptr, "neighbor_histogram_batched: null pointer");
    HistStages st;
    long long max_rows = 0;
    for (int s = 0; s < (int)num_stages; ++s) {
        GEOB_REQUIRE(neighbors[s] != nullptr && widths[s] >= 1 && widths[s] <= (1 << 20),
                     "neighbor_histogram_batched: stage %d has no table or a bad width", s);
        long long row = 0;
        for (int c = 0; c < 2 * (int)batch; ++c) {
            GEOB_REQUIRE(cloud_rows[s * 2 * batch + c] >= 1, "neighbor_histogram_batched: stage %d cloud %d is empty", s, c);
            st.cloud_start[s][c] = (int)row;
            row += cloud_rows[s * 2 * batch + c];
            GEOB_REQUIRE(row < (1LL << 31), "neighbor_histogram_batched: stage %d has 2^31 rows or more", s);
        }
        st.cloud_start[s][2 * batch] = (int)row;
        st.nbr[s] = (const long long*)neighbors[s];
        st.rows[s] = row;
        st.width[s] = (int)widths[s];
        max_rows = row > max_rows ? row : max_rows;
    }
    cudaStream_t cs = (cudaStream_t)stream;
    GEOB_CHECK_CUDA(cudaMemsetAsync(hists, 0, sizeof(int32_t) * (size_t)batch * num_stages * hist_n, cs));
    neighbor_histogram_batched_kernel<<<dim3((unsigned)((max_rows + 255) / 256), (unsigned)num_stages), 256, 0, cs>>>(
        st, (int)num_stages, (int)batch, (int)hist_n, hists);
    neighbor_histogram_stop_kernel<<<1, 256, 0, cs>>>(hists, (int)num_stages, (int)batch, (int)hist_n, (long long)sample_threshold,
                                                      totals, stop);
    GEOB_CHECK_LAUNCH();
    count_launches(2);
    return 0;
}

}  // extern "C"
