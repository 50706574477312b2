// Voxel downsampling with Open3D's semantics (PointCloud::VoxelDownSample), batched over up to 64 clouds.
//
// Contract (DESIGN.md section 8a), all arithmetic in IEEE double with no FMA contraction:
//   lo = min_i p_i - 0.5 v, hi = max_i p_i + 0.5 v (componentwise); error if v * INT_MAX < max(hi - lo) (Open3D's "voxel_size is
//   too small"), on a non-finite coordinate, or when an axis spans 2^21 voxels or more (the packed key's limit);
//   voxel of point i: k_a = int(floor((p_i[a] - lo[a]) / v));
//   value of a voxel: the double sum of its points in INPUT order, divided by double(count) (normals likewise, not renormalised);
//   output order: iteration order of a default-constructed std::unordered_map<Vector3i, ...> filled by operator[] in input order,
//   hashed by Open3D's hash_eigen (seed = 0; seed ^= size_t(k) + 0x9e3779b9 + (seed << 6) + (seed >> 2) for x, y, z).
//
// Stages: bounds and checks (one CTA per cloud) -> packed voxel key per point and an open-addressing table that records each
// voxel's first point -> first-occurrence ranks (per-cloud scan) -> hash_eigen of each voxel -> a stable LSD radix sort of the
// points by voxel, which lists every voxel's points in input order in linear time -> sequential double sums per voxel -> the
// libstdc++ order (unordered_map.cuh) and the gather.  Data-dependent errors go to a status word after the lengths, so the
// caller learns of them with the one read-back of the lengths.
#include <math.h>

#include "common.cuh"
#include "geob200.h"
#include "unordered_map.cuh"

namespace geob200 {

namespace {

constexpr int kAxisBits = 21;                   // a voxel key packs three 21-bit axis indices
constexpr int kRadixTile = 2048;                // items per CTA of a radix pass (256 threads x 8 rounds)
constexpr unsigned long long kEmpty = 0xFFFFFFFFFFFFFFFFull;

struct VxCloud {
    double lo[3];
};

__device__ __forceinline__ void set_status(int* status, int code) { atomicCAS(status, 0, code); }

// min / max in double, the finiteness check, lo, the too-small check and the axis limit
__global__ void __launch_bounds__(1024) vx_bounds_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs, double voxel,
                                                         VxCloud* __restrict__ out, int* __restrict__ status) {
    const CloudSeg sg = segs[blockIdx.x];
    double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    bool finite = true;
    for (int i = threadIdx.x; i < sg.len; i += blockDim.x) {
        const double* p = pts + 3ll * (sg.start + i);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double x = p[a];
            finite = finite && isfinite(x);
            mn[a] = fmin(mn[a], x);
            mx[a] = fmax(mx[a], x);
        }
    }
    if (__syncthreads_or(!finite)) {
        if (threadIdx.x == 0) set_status(status, GEOB200_VOXEL_NONFINITE);
        return;
    }
    __shared__ double smn[3][32], smx[3][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmax(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if (lane == 0) { smn[a][warp] = mn[a]; smx[a][warp] = mx[a]; }
    }
    __syncthreads();
    if (threadIdx.x == 0 && sg.len > 0) {
        const int nw = blockDim.x >> 5;
        VxCloud c;
        double extent = 0.0;
        const double half = 0.5 * voxel;   // exact
        bool axis_ok = true;
        for (int a = 0; a < 3; ++a) {
            double lo = smn[a][0], hi = smx[a][0];
            for (int w = 1; w < nw; ++w) { lo = fmin(lo, smn[a][w]); hi = fmax(hi, smx[a][w]); }
            const double vlo = __dsub_rn(lo, half), vhi = __dadd_rn(hi, half);
            extent = fmax(extent, __dsub_rn(vhi, vlo));
            c.lo[a] = vlo;
            // floor and IEEE subtraction / division are monotone, so the largest index of the axis is the maximum's
            axis_ok = axis_ok && floor(__ddiv_rn(__dsub_rn(hi, vlo), voxel)) < (double)(1 << kAxisBits);
        }
        out[blockIdx.x] = c;
        if (__dmul_rn(voxel, 2147483647.0) < extent) set_status(status, GEOB200_VOXEL_TOO_SMALL);
        else if (!axis_ok) set_status(status, GEOB200_VOXEL_AXIS_LIMIT);
    }
}

__device__ __forceinline__ void voxel_index(const double* p, const VxCloud& c, double voxel, int k[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) k[a] = (int)floor(__ddiv_rn(__dsub_rn(p[a], c.lo[a]), voxel));
}

__device__ __forceinline__ unsigned long long pack_key(const int k[3]) {
    return (unsigned long long)k[0] | ((unsigned long long)k[1] << kAxisBits) | ((unsigned long long)k[2] << (2 * kAxisBits));
}

// Open3D's utility::hash_eigen<Eigen::Vector3i>; std::hash<int> is the identity cast to size_t
__device__ __forceinline__ unsigned long long hash_eigen(const int k[3]) {
    unsigned long long seed = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) seed ^= (unsigned long long)(long long)k[a] + 0x9e3779b9ull + (seed << 6) + (seed >> 2);
    return seed;
}

// packed key per point and its slot in the cloud's open-addressing table (2 len slots), which keeps each voxel's first point
__global__ void vx_insert_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs, const VxCloud* __restrict__ clouds,
                                 double voxel, const int* __restrict__ status, unsigned long long* __restrict__ tab_key,
                                 int* __restrict__ tab_first, int* __restrict__ pt_slot) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    int k[3];
    voxel_index(pts + 3ll * (sg.start + i), clouds[blockIdx.y], voxel, k);
    const unsigned long long key = pack_key(k);
    const unsigned tsize = 2u * (unsigned)sg.len;
    const long long tbase = 2ll * sg.start;
    unsigned h = (unsigned)(mix64(key) % tsize);
    while (true) {
        const unsigned long long prev = atomicCAS(&tab_key[tbase + h], kEmpty, key);
        if (prev == kEmpty || prev == key) break;
        h = (h + 1 == tsize) ? 0 : h + 1;
    }
    atomicMin(&tab_first[tbase + h], i);
    pt_slot[sg.start + i] = (int)h;
}

__global__ void vx_flag_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ status, const int* __restrict__ tab_first,
                               const int* __restrict__ pt_slot, int* __restrict__ flag) {
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    flag[sg.start + i] = (*status == 0 && tab_first[2ll * sg.start + pt_slot[sg.start + i]] == i) ? 1 : 0;
}

// voxel offsets per cloud; out_lengths[b] = voxels of cloud b (0 on error), out_lengths[batch] = the status word
__global__ void vx_offsets_kernel(const int* __restrict__ m, int nb, const int* __restrict__ status, int* __restrict__ voff,
                                  long long* __restrict__ out_lengths) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        const int st = *status;
        int acc = 0;
        for (int b = 0; b < nb; ++b) {
            voff[b] = acc;
            const int mb = st ? 0 : m[b];
            acc += mb;
            out_lengths[b] = mb;
        }
        voff[nb] = acc;
        out_lengths[nb] = st;
    }
}

// first points: the slot's voxel id G = voff + rank and hash_eigen of the voxel
__global__ void vx_setup_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs, const VxCloud* __restrict__ clouds,
                                double voxel, const int* __restrict__ status, const int* __restrict__ flag, const int* __restrict__ rank,
                                const int* __restrict__ voff, const int* __restrict__ pt_slot, int* __restrict__ tab_vox,
                                unsigned long long* __restrict__ vox_hash) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len || !flag[sg.start + i]) return;
    int k[3];
    voxel_index(pts + 3ll * (sg.start + i), clouds[blockIdx.y], voxel, k);
    const int G = voff[blockIdx.y] + rank[sg.start + i];
    tab_vox[2ll * sg.start + pt_slot[sg.start + i]] = G;
    vox_hash[G] = hash_eigen(k);
}

// radix-sort items: key = voxel id of the point, value = its stacked row
__global__ void vx_keys_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ status, const int* __restrict__ tab_vox,
                               const int* __restrict__ pt_slot, int* __restrict__ key, int* __restrict__ val) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    key[sg.start + i] = tab_vox[2ll * sg.start + pt_slot[sg.start + i]];
    val[sg.start + i] = sg.start + i;
}

// ---- stable LSD radix sort, 8-bit digits: tile histograms, digit-major scan, stable scatter ----

__global__ void __launch_bounds__(256) vx_radix_hist_kernel(const int* __restrict__ key, int n, int shift, int ntiles,
                                                            const int* __restrict__ status, int* __restrict__ hist) {
    if (*status) return;
    __shared__ int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int base = blockIdx.x * kRadixTile;
    for (int r = 0; r < kRadixTile / 256; ++r) {
        const int p = base + r * 256 + threadIdx.x;
        if (p < n) atomicAdd(&h[(key[p] >> shift) & 255], 1);
    }
    __syncthreads();
    hist[threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];   // digit-major: the scan runs digit by digit
}

__global__ void vx_digit_segs_kernel(int ntiles, CloudSeg* __restrict__ dsegs) {
    const int d = threadIdx.x;
    dsegs[d].start = d * ntiles;
    dsegs[d].len = ntiles;
}

// Items of a tile go in rounds of 256 (item order = round, warp, lane); within a round a warp ranks equal digits with
// __match_any_sync, and the per-warp digit counts of the round give each warp's offset.  Every item lands after all earlier
// items of its digit: the pass is stable.
__global__ void __launch_bounds__(256) vx_radix_scatter_kernel(const int* __restrict__ key_in, const int* __restrict__ val_in, int n,
                                                               int shift, int ntiles, const int* __restrict__ status,
                                                               const int* __restrict__ hist_scan, const int* __restrict__ digit_tot,
                                                               int* __restrict__ key_out, int* __restrict__ val_out) {
    if (*status) return;
    __shared__ int run[256];          // next output position of each digit in this tile
    __shared__ int wcnt[8][256];      // per-warp digit counts of the current round
    __shared__ int dbase[256];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    // exclusive scan of the digit totals (256 values, one warp)
    if (warp == 0) {
        int v[8], s = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) { v[j] = digit_tot[lane * 8 + j]; s += v[j]; }
        int x = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        int e = x - s;
#pragma unroll
        for (int j = 0; j < 8; ++j) { dbase[lane * 8 + j] = e; e += v[j]; }
    }
    __syncthreads();
    run[t] = dbase[t] + hist_scan[t * ntiles + blockIdx.x];
    const int base = blockIdx.x * kRadixTile;
    for (int r = 0; r < kRadixTile / 256; ++r) {
#pragma unroll
        for (int w = 0; w < 8; ++w) wcnt[w][t] = 0;
        __syncthreads();
        const int p = base + r * 256 + t;
        const bool valid = p < n;
        const int k = valid ? key_in[p] : 0;
        const int d = valid ? (k >> shift) & 255 : 256;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int lrank = __popc(peers & ((1u << lane) - 1u));
        if (valid && lrank == 0) wcnt[warp][d] = __popc(peers);
        __syncthreads();
        if (valid) {
            int off = run[d] + lrank;
            for (int w = 0; w < warp; ++w) off += wcnt[w][d];
            key_out[off] = k;
            val_out[off] = val_in[p];
        }
        __syncthreads();
        int add = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) add += wcnt[w][t];
        run[t] += add;
        __syncthreads();
    }
}

// start of every voxel's run in the sorted order (keys are the voxel ids 0..M-1, each present)
__global__ void vx_starts_kernel(const int* __restrict__ key, int n, const int* __restrict__ status, int* __restrict__ vox_start) {
    if (*status) return;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    if (p == 0 || key[p] != key[p - 1]) vox_start[key[p]] = p;
}

// sequential double sums in input order, divided by double(count) (AccumulatedPoint::GetAveragePoint / GetAverageNormal)
__global__ void vx_sum_kernel(const double* __restrict__ pts, const double* __restrict__ nrm, int n, const int* __restrict__ status,
                              const int* __restrict__ voff, int nb, const int* __restrict__ vox_start, const int* __restrict__ sorted_val,
                              double* __restrict__ vox_pts, double* __restrict__ vox_nrm) {
    if (*status) return;
    const int G = blockIdx.x * blockDim.x + threadIdx.x;
    const int M = voff[nb];
    if (G >= M) return;
    const int s = vox_start[G], e = (G + 1 < M) ? vox_start[G + 1] : n;
    double sx = 0.0, sy = 0.0, sz = 0.0, nx = 0.0, ny = 0.0, nz = 0.0;
#pragma unroll 4
    for (int q = s; q < e; ++q) {
        const long long row = sorted_val[q];
        const double* p = pts + 3 * row;
        sx = __dadd_rn(sx, p[0]);
        sy = __dadd_rn(sy, p[1]);
        sz = __dadd_rn(sz, p[2]);
        if (nrm != nullptr) {
            const double* m = nrm + 3 * row;
            nx = __dadd_rn(nx, m[0]);
            ny = __dadd_rn(ny, m[1]);
            nz = __dadd_rn(nz, m[2]);
        }
    }
    const double c = (double)(e - s);
    vox_pts[3ll * G + 0] = __ddiv_rn(sx, c);
    vox_pts[3ll * G + 1] = __ddiv_rn(sy, c);
    vox_pts[3ll * G + 2] = __ddiv_rn(sz, c);
    if (nrm != nullptr) {
        vox_nrm[3ll * G + 0] = __ddiv_rn(nx, c);
        vox_nrm[3ll * G + 1] = __ddiv_rn(ny, c);
        vox_nrm[3ll * G + 2] = __ddiv_rn(nz, c);
    }
}

// one CTA per cloud: the unordered_map order of its voxels under hash_eigen, then the gather of points (and normals)
__global__ void __launch_bounds__(1024) vx_order_kernel(const CloudSeg* __restrict__ segs, const int* __restrict__ status,
                                                        const int* __restrict__ voff, const unsigned long long* __restrict__ vox_hash,
                                                        const double* __restrict__ vox_pts, const double* __restrict__ vox_nrm,
                                                        int* __restrict__ cur_g, int* __restrict__ nxt_g, int* __restrict__ A_g,
                                                        int* __restrict__ lnk_g, int* __restrict__ bucket_scratch,
                                                        double* __restrict__ out_pts, double* __restrict__ out_nrm) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.x];
    const int v0 = voff[blockIdx.x];
    const int m = voff[blockIdx.x + 1] - v0;
    int* act = bucket_scratch + (3ll * sg.start + 64ll * blockIdx.x) * 3;
    const long long bcap = 3ll * sg.len + 64;
    const int* order = unordered_map_order(m, vox_hash + v0, cur_g + sg.start, nxt_g + sg.start, A_g + sg.start, lnk_g + sg.start,
                                           act, act + bcap, act + 2 * bcap);
    for (int q = threadIdx.x; q < 3 * m; q += blockDim.x) {
        const long long src = 3ll * (v0 + order[q / 3]) + q % 3;
        out_pts[3ll * v0 + q] = vox_pts[src];
        if (out_nrm != nullptr) out_nrm[3ll * v0 + q] = vox_nrm[src];
    }
}

int radix_passes(int64_t n_points) {
    int bits = 0;
    while (bits < 31 && (1ll << bits) < n_points) ++bits;   // voxel ids are < n_points
    return bits <= 8 ? 1 : (bits + 7) / 8;
}

}  // namespace

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_voxel_down_sample_workspace_bytes(int64_t n_points, int64_t batch) {
    if (n_points < 0 || batch < 0) return 0;
    const size_t n = (size_t)n_points, b = (size_t)batch;
    const size_t ntiles = (n + kRadixTile - 1) / kRadixTile;
    size_t bytes = 0;
    bytes += align_up(sizeof(CloudSeg) * b, 256) + align_up(sizeof(VxCloud) * b, 256) + align_up(sizeof(CloudSeg) * 256, 256);
    bytes += align_up(8 * 2 * n, 256) + align_up(4 * 2 * n, 256) * 2;   // tab_key, tab_first, tab_vox
    bytes += align_up(4 * n, 256) * 12;                                 // slot, flag, rank, keys x2, vals x2, start, cur, nxt, A, lnk
    bytes += align_up(8 * n, 256);                                      // vox_hash
    bytes += align_up(8 * 3 * n, 256) * 2;                              // vox_pts, vox_nrm
    bytes += align_up(4 * 256 * ntiles, 256) + align_up(4 * 256, 256);  // tile histograms, digit totals
    bytes += align_up(4 * 3 * (3 * n + 64 * b), 256);                   // bucket scratch
    bytes += align_up(4 * (b + 1), 256) * 2 + 256;                      // m_per_cloud, voff, status
    return bytes + 4096;
}

int geob200_voxel_down_sample(const double* points, const double* normals, int64_t n_points, const int64_t* lengths_h, int64_t batch,
                              double voxel, double* out_points, double* out_normals, int64_t* out_lengths, void* workspace,
                              size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(batch >= 1 && batch <= GEOB200_VOXEL_MAX_CLOUDS, "voxel_down_sample: batch must be in 1..%d, got %lld",
                 GEOB200_VOXEL_MAX_CLOUDS, (long long)batch);
    GEOB_REQUIRE(lengths_h != nullptr && out_lengths != nullptr, "voxel_down_sample: null lengths pointer");
    GEOB_REQUIRE(n_points >= 0 && n_points < (1ll << 30), "voxel_down_sample: n_points must be in 0..2^30-1, got %lld",
                 (long long)n_points);
    GEOB_REQUIRE(voxel > 0.0 && isfinite(voxel), "voxel_down_sample: voxel size must be positive and finite, got %g", voxel);
    int64_t total = 0;
    int max_len = 0;
    for (int64_t b = 0; b < batch; ++b) {
        GEOB_REQUIRE(lengths_h[b] >= 0, "voxel_down_sample: cloud %lld has a negative length", (long long)b);
        total += lengths_h[b];
        if (lengths_h[b] > max_len) max_len = (int)lengths_h[b];
    }
    GEOB_REQUIRE(total == n_points, "voxel_down_sample: sum(lengths)=%lld != n_points=%lld", (long long)total, (long long)n_points);
    GEOB_REQUIRE(n_points == 0 || (points != nullptr && out_points != nullptr), "voxel_down_sample: null point pointer");
    GEOB_REQUIRE((normals == nullptr) == (out_normals == nullptr), "voxel_down_sample: normals and out_normals must both be given or both be null");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_voxel_down_sample_workspace_bytes(n_points, batch),
                 "voxel_down_sample: workspace too small (%zu bytes, need %zu)", workspace_bytes,
                 geob200_voxel_down_sample_workspace_bytes(n_points, batch));

    Arena ar(workspace, workspace_bytes);
    const size_t n = (size_t)n_points;
    const int ntiles = (int)((n + kRadixTile - 1) / kRadixTile);
    CloudSeg* segs = ar.take<CloudSeg>(batch);
    VxCloud* clouds = ar.take<VxCloud>(batch);
    CloudSeg* dsegs = ar.take<CloudSeg>(256);
    unsigned long long* tab_key = ar.take<unsigned long long>(2 * n);
    int* tab_first = ar.take<int>(2 * n);
    int* tab_vox = ar.take<int>(2 * n);
    int* pt_slot = ar.take<int>(n);
    int* flag = ar.take<int>(n);
    int* rank = ar.take<int>(n);
    int* key[2] = {ar.take<int>(n), ar.take<int>(n)};
    int* val[2] = {ar.take<int>(n), ar.take<int>(n)};
    int* vox_start = ar.take<int>(n);
    int* cur = ar.take<int>(n);
    int* nxt = ar.take<int>(n);
    int* A = ar.take<int>(n);
    int* lnk = ar.take<int>(n);
    unsigned long long* vox_hash = ar.take<unsigned long long>(n);
    double* vox_pts = ar.take<double>(3 * n);
    double* vox_nrm = ar.take<double>(3 * n);
    int* hist = ar.take<int>(256 * (size_t)ntiles);
    int* digit_tot = ar.take<int>(256);
    int* bucket_scratch = ar.take<int>(3 * (3 * n + 64 * (size_t)batch));
    int* m_per_cloud = ar.take<int>(batch + 1);
    int* voff = ar.take<int>(batch + 1);
    int* status = ar.take<int>(64);
    GEOB_REQUIRE(ar.ok(), "voxel_down_sample: workspace accounting error");

    CloudSeg h[GEOB200_VOXEL_MAX_CLOUDS];
    for (int64_t b = 0, acc = 0; b < batch; acc += lengths_h[b], ++b) {
        h[b].start = (int)acc;
        h[b].len = (int)lengths_h[b];
    }
    GEOB_CHECK_CUDA(cudaMemcpyAsync(segs, h, sizeof(CloudSeg) * batch, cudaMemcpyHostToDevice, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
    if (n == 0) {   // only empty clouds: every length is zero, no launch
        GEOB_CHECK_CUDA(cudaMemsetAsync(out_lengths, 0, sizeof(int64_t) * (batch + 1), st));
        return 0;
    }
    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_key, 0xFF, 8 * 2 * n, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_first, 0x7F, 4 * 2 * n, st));

    const unsigned nbt = (unsigned)batch;
    const dim3 pgrid((max_len + 255) / 256, nbt);
    vx_bounds_kernel<<<nbt, 1024, 0, st>>>(points, segs, voxel, clouds, status);
    vx_insert_kernel<<<pgrid, 256, 0, st>>>(points, segs, clouds, voxel, status, tab_key, tab_first, pt_slot);
    vx_flag_kernel<<<pgrid, 256, 0, st>>>(segs, status, tab_first, pt_slot, flag);
    seg_exclusive_scan_kernel<<<nbt, 1024, 0, st>>>(flag, rank, segs, m_per_cloud);
    vx_offsets_kernel<<<1, 32, 0, st>>>(m_per_cloud, (int)batch, status, voff, (long long*)out_lengths);
    vx_setup_kernel<<<pgrid, 256, 0, st>>>(points, segs, clouds, voxel, status, flag, rank, voff, pt_slot, tab_vox, vox_hash);
    vx_keys_kernel<<<pgrid, 256, 0, st>>>(segs, status, tab_vox, pt_slot, key[0], val[0]);
    vx_digit_segs_kernel<<<1, 256, 0, st>>>(ntiles, dsegs);
    const int passes = radix_passes(n_points);
    for (int pass = 0; pass < passes; ++pass) {
        const int in = pass & 1, shift = 8 * pass;
        vx_radix_hist_kernel<<<ntiles, 256, 0, st>>>(key[in], (int)n, shift, ntiles, status, hist);
        seg_exclusive_scan_kernel<<<256, 1024, 0, st>>>(hist, hist, dsegs, digit_tot);
        vx_radix_scatter_kernel<<<ntiles, 256, 0, st>>>(key[in], val[in], (int)n, shift, ntiles, status, hist, digit_tot, key[in ^ 1],
                                                        val[in ^ 1]);
    }
    const int fin = passes & 1;
    vx_starts_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(key[fin], (int)n, status, vox_start);
    vx_sum_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(points, normals, (int)n, status, voff, (int)batch, vox_start, val[fin],
                                                                vox_pts, vox_nrm);
    vx_order_kernel<<<nbt, 1024, 0, st>>>(segs, status, voff, vox_hash, vox_pts, vox_nrm, cur, nxt, A, lnk, bucket_scratch, out_points,
                                         out_normals);
    GEOB_CHECK_LAUNCH();
    count_launches(11 + 3 * passes);
    return 0;
}

}  // extern "C"
