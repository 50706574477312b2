// Normal estimation with Open3D's semantics (PointCloud::EstimateNormals with FastEigen3x3), batched over up to 64 clouds,
// and the reference's regularize_normals.
//
// Contract (DESIGN.md section 8a), all arithmetic in IEEE double with no FMA contraction:
//   neighbours of p_i: the min(knn, N) points nearest to it (itself included), or with a radius those with d2 < radius^2, capped at
//   knn; d2 = ((dx dx) + dy dy) + dz dz; ascending (d2, index);
//   cumulants x, y, z, xx, xy, xz, yy, yz, zz summed over the neighbours in that order, each divided by the count; the covariance
//   entry ab is E[ab] - E[a] E[b];
//   normal: FastEigen3x3 (Eberly's robust symmetric 3x3 eigensolver) of the covariance, the unit eigenvector of its smallest
//   eigenvalue, signed as the construction gives it; (0, 0, 1) for fewer than 3 neighbours or a zero-norm result.
//
// Stages: bounds, finiteness and the grid's cell size (one CTA per cloud) -> packed cell key per point in an open-addressing table
// (the voxel tables' layout: 2 len slots per cloud) with a point count per cell -> per-cloud scan of the counts -> points scattered
// into cell order -> one warp per query: exact kNN ring by ring over the hashed cells with the top-k in registers, then the
// cumulants and the eigensolver.  A non-finite coordinate goes to the status word; no output is written then.
#include <math.h>

#include "common.cuh"
#include "geob200.h"
#include "unordered_map.cuh"

namespace geob200 {

namespace {

constexpr int kAxisBits = 21;
constexpr int kMaxAxisCells = 1 << 20;          // cells per axis stay below this, so ring indices never leave 21 bits
constexpr unsigned long long kEmpty = 0xFFFFFFFFFFFFFFFFull;

struct NmCloud {
    double lo[3];
    double h;           // cell edge
    double slack;       // what rounding may take off a ring's distance bound (see nm_knn_kernel)
    int dims[3];        // cells per axis
};

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

// bounds and finiteness in double, then the cell edge: about max(knn, 8) / 2 points per cell on a surface that fills the bounding
// box's faces, or along a line; never more than 2^20 cells per axis
__global__ void __launch_bounds__(1024) nm_bounds_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs, int knn,
                                                         double radius, NmCloud* __restrict__ out, int* __restrict__ status) {
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
        if (threadIdx.x == 0) atomicCAS(status, 0, GEOB200_NORMALS_NONFINITE);
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
    if (threadIdx.x != 0 || sg.len == 0) return;
    const int nw = blockDim.x >> 5;
    NmCloud c;
    double ext[3], emax = 0.0, amax = 0.0;
    for (int a = 0; a < 3; ++a) {
        double lo = smn[a][0], hi = smx[a][0];
        for (int w = 1; w < nw; ++w) { lo = fmin(lo, smn[a][w]); hi = fmax(hi, smx[a][w]); }
        c.lo[a] = lo;
        ext[a] = hi - lo;
        emax = fmax(emax, ext[a]);
        amax = fmax(amax, fmax(fabs(lo), fabs(hi)));
    }
    const double per_cell = 0.5 * (double)(knn > 8 ? knn : 8), n = (double)sg.len;
    const double area = ext[0] * ext[1] + ext[0] * ext[2] + ext[1] * ext[2];
    double h = fmax(sqrt(area * per_cell / n), emax * per_cell / n);
    if (radius > 0.0) h = fmin(h, radius);
    h = fmax(h, emax * (1.0 + 1e-6) / (double)(kMaxAxisCells - 2));
    if (!(h > 0.0) || !isfinite(h)) h = 1.0;          // all points coincide
    c.h = h;
    // cell indices are floor(fl(fl(p - lo) / h)): each of the two roundings moves a boundary by at most 2^-53 of (|p| + extent)
    c.slack = 1e-12 * (amax + emax + h);
    for (int a = 0; a < 3; ++a) c.dims[a] = (int)floor(dd(ext[a], h)) + 1;
    out[blockIdx.x] = c;
}

__device__ __forceinline__ int cell_of(double x, double lo, double h) { return (int)floor(dd(ds(x, lo), h)); }

__device__ __forceinline__ unsigned long long pack_cell(int x, int y, int z) {
    return (unsigned long long)x | ((unsigned long long)y << kAxisBits) | ((unsigned long long)z << (2 * kAxisBits));
}

// cell key per point, its slot in the cloud's table (2 len slots) and the cell's point count
__global__ void nm_insert_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs, const NmCloud* __restrict__ clouds,
                                 const int* __restrict__ status, unsigned long long* __restrict__ tab_key, int* __restrict__ tab_cnt,
                                 int* __restrict__ pt_slot) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const NmCloud c = clouds[blockIdx.y];
    const double* p = pts + 3ll * (sg.start + i);
    const unsigned long long key = pack_cell(cell_of(p[0], c.lo[0], c.h), cell_of(p[1], c.lo[1], c.h), cell_of(p[2], c.lo[2], c.h));
    const unsigned tsize = 2u * (unsigned)sg.len;
    const long long tbase = 2ll * sg.start;
    unsigned h = (unsigned)(mix64(key) % tsize);
    while (true) {
        const unsigned long long prev = atomicCAS(&tab_key[tbase + h], kEmpty, key);
        if (prev == kEmpty || prev == key) break;
        h = (h + 1 == tsize) ? 0 : h + 1;
    }
    atomicAdd(&tab_cnt[tbase + h], 1);
    pt_slot[sg.start + i] = (int)h;
}

// points into cell order: the cell's start (scan of the counts) plus an arrival rank.  The order inside a cell is not fixed, and
// nothing depends on it: the search keeps the exact top-k under the total order (d2, index).
__global__ void nm_scatter_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs, const int* __restrict__ status,
                                  const int* __restrict__ pt_slot, const int* __restrict__ tab_start, int* __restrict__ tab_fill,
                                  double* __restrict__ sorted_xyz, int* __restrict__ sorted_idx) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.len) return;
    const long long slot = 2ll * sg.start + pt_slot[sg.start + i];
    const long long q = sg.start + tab_start[slot] + atomicAdd(&tab_fill[slot], 1);
    const double* p = pts + 3ll * (sg.start + i);
    sorted_xyz[3 * q + 0] = p[0];
    sorted_xyz[3 * q + 1] = p[1];
    sorted_xyz[3 * q + 2] = p[2];
    sorted_idx[q] = i;
}

struct V3 {
    double x, y, z;
};
__device__ __forceinline__ V3 cross(const V3& a, const V3& b) {
    return {ds(dm(a.y, b.z), dm(a.z, b.y)), ds(dm(a.z, b.x), dm(a.x, b.z)), ds(dm(a.x, b.y), dm(a.y, b.x))};
}
// Eigen 3.3's 3-vector dot: one two-double packet and the third product, (a0 b0 + a1 b1) + a2 b2
__device__ __forceinline__ double dot(const V3& a, const V3& b) { return da(da(dm(a.x, b.x), dm(a.y, b.y)), dm(a.z, b.z)); }
__device__ __forceinline__ V3 vdiv(const V3& a, double s) { return {dd(a.x, s), dd(a.y, s), dd(a.z, s)}; }

// A: a00 a01 a02 a11 a12 a22 (symmetric)
struct Sym3 {
    double a00, a01, a02, a11, a12, a22;
};

__device__ V3 eigenvector0(const Sym3& A, double ev) {
    const V3 r0 = {ds(A.a00, ev), A.a01, A.a02}, r1 = {A.a01, ds(A.a11, ev), A.a12}, r2 = {A.a02, A.a12, ds(A.a22, ev)};
    const V3 r0xr1 = cross(r0, r1), r0xr2 = cross(r0, r2), r1xr2 = cross(r1, r2);
    const double d0 = dot(r0xr1, r0xr1), d1 = dot(r0xr2, r0xr2), d2 = dot(r1xr2, r1xr2);
    double dmax = d0;
    int imax = 0;
    if (d1 > dmax) { dmax = d1; imax = 1; }
    if (d2 > dmax) imax = 2;
    if (imax == 0) return vdiv(r0xr1, sqrt(d0));
    if (imax == 1) return vdiv(r0xr2, sqrt(d1));
    return vdiv(r1xr2, sqrt(d2));
}

__device__ V3 eigenvector1(const Sym3& A, const V3& e0, double ev) {
    V3 U;
    if (fabs(e0.x) > fabs(e0.y)) {
        const double inv = dd(1.0, sqrt(da(dm(e0.x, e0.x), dm(e0.z, e0.z))));
        U = {dm(-e0.z, inv), 0.0, dm(e0.x, inv)};
    } else {
        const double inv = dd(1.0, sqrt(da(dm(e0.y, e0.y), dm(e0.z, e0.z))));
        U = {0.0, dm(e0.z, inv), dm(-e0.y, inv)};
    }
    const V3 V = cross(e0, U);
    const V3 AU = {da(da(dm(A.a00, U.x), dm(A.a01, U.y)), dm(A.a02, U.z)), da(da(dm(A.a01, U.x), dm(A.a11, U.y)), dm(A.a12, U.z)),
                   da(da(dm(A.a02, U.x), dm(A.a12, U.y)), dm(A.a22, U.z))};
    const V3 AV = {da(da(dm(A.a00, V.x), dm(A.a01, V.y)), dm(A.a02, V.z)), da(da(dm(A.a01, V.x), dm(A.a11, V.y)), dm(A.a12, V.z)),
                   da(da(dm(A.a02, V.x), dm(A.a12, V.y)), dm(A.a22, V.z))};
    double m00 = ds(da(da(dm(U.x, AU.x), dm(U.y, AU.y)), dm(U.z, AU.z)), ev);
    double m01 = da(da(dm(U.x, AV.x), dm(U.y, AV.y)), dm(U.z, AV.z));
    double m11 = ds(da(da(dm(V.x, AV.x), dm(V.y, AV.y)), dm(V.z, AV.z)), ev);
    const double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
    if (a00 >= a11) {
        if (fmax(a00, a01) > 0.0) {
            if (a00 >= a01) {
                m01 = dd(m01, m00);
                m00 = dd(1.0, sqrt(da(1.0, dm(m01, m01))));
                m01 = dm(m01, m00);
            } else {
                m00 = dd(m00, m01);
                m01 = dd(1.0, sqrt(da(1.0, dm(m00, m00))));
                m00 = dm(m00, m01);
            }
            return {ds(dm(m01, U.x), dm(m00, V.x)), ds(dm(m01, U.y), dm(m00, V.y)), ds(dm(m01, U.z), dm(m00, V.z))};
        }
        return U;
    }
    if (fmax(a11, a01) > 0.0) {
        if (a11 >= a01) {
            m01 = dd(m01, m11);
            m11 = dd(1.0, sqrt(da(1.0, dm(m01, m01))));
            m01 = dm(m01, m11);
        } else {
            m11 = dd(m11, m01);
            m01 = dd(1.0, sqrt(da(1.0, dm(m11, m11))));
            m11 = dm(m11, m01);
        }
        return {ds(dm(m11, U.x), dm(m01, V.x)), ds(dm(m11, U.y), dm(m01, V.y)), ds(dm(m11, U.z), dm(m01, V.z))};
    }
    return U;
}

// Open3D's FastEigen3x3: the eigenvector of the smallest eigenvalue (zero when the largest coefficient is 0)
__device__ V3 fast_eigen3x3(Sym3 A) {
    const double maxc = fmax(fmax(fmax(A.a00, A.a01), fmax(A.a02, A.a11)), fmax(A.a12, A.a22));
    if (maxc == 0.0) return {0.0, 0.0, 0.0};
    const Sym3 S = {dd(A.a00, maxc), dd(A.a01, maxc), dd(A.a02, maxc), dd(A.a11, maxc), dd(A.a12, maxc), dd(A.a22, maxc)};
    const double norm = da(da(dm(S.a01, S.a01), dm(S.a02, S.a02)), dm(S.a12, S.a12));
    if (norm > 0.0) {
        const double q = dd(da(da(S.a00, S.a11), S.a22), 3.0);
        const double b00 = ds(S.a00, q), b11 = ds(S.a11, q), b22 = ds(S.a22, q);
        const double p = sqrt(dd(da(da(da(dm(b00, b00), dm(b11, b11)), dm(b22, b22)), dm(norm, 2.0)), 6.0));
        const double c00 = ds(dm(b11, b22), dm(S.a12, S.a12));
        const double c01 = ds(dm(S.a01, b22), dm(S.a12, S.a02));
        const double c02 = ds(dm(S.a01, S.a12), dm(b11, S.a02));
        const double det = dd(da(ds(dm(b00, c00), dm(S.a01, c01)), dm(S.a02, c02)), dm(dm(p, p), p));
        const double half_det = fmin(fmax(dm(det, 0.5), -1.0), 1.0);
        const double angle = dd(acos(half_det), 3.0);
        const double two_thirds_pi = 2.09439510239319549;
        const double beta2 = dm(cos(angle), 2.0);
        const double beta0 = dm(cos(da(angle, two_thirds_pi)), 2.0);
        const double beta1 = -da(beta0, beta2);
        const double ev0 = da(q, dm(p, beta0)), ev1 = da(q, dm(p, beta1)), ev2 = da(q, dm(p, beta2));
        if (half_det >= 0.0) {
            const V3 e2 = eigenvector0(S, ev2);
            if (ev2 < ev0 && ev2 < ev1) return e2;
            const V3 e1 = eigenvector1(S, e2, ev1);
            if (ev1 < ev0 && ev1 < ev2) return e1;
            return cross(e1, e2);
        }
        const V3 e0 = eigenvector0(S, ev0);
        if (ev0 < ev1 && ev0 < ev2) return e0;
        const V3 e1 = eigenvector1(S, e0, ev1);
        if (ev1 < ev0 && ev1 < ev2) return e1;
        return cross(e0, e1);
    }
    // diagonal: Open3D compares the entries after A /= maxc; A *= maxc, which need not give A back
    const double d0 = dm(S.a00, maxc), d1 = dm(S.a11, maxc), d2 = dm(S.a22, maxc);
    if (d0 < d1 && d0 < d2) return {1.0, 0.0, 0.0};
    if (d1 < d0 && d1 < d2) return {0.0, 1.0, 0.0};
    return {0.0, 0.0, 1.0};
}

// (d2, index) lexicographic
__device__ __forceinline__ bool before(double da_, int ia, double db_, int ib) { return da_ < db_ || (da_ == db_ && ia < ib); }

// One warp per query (queries in cell order, so the warps of a CTA search neighbouring cells).  Rings of cells at Chebyshev
// distance r = 0, 1, 2, ... around the query's cell are scanned; each cell's points are read by the lanes, and candidates that beat
// the current k-th entry go one at a time into the warp's sorted top-k (entry j in lane j & 31, register j >> 5).  After ring r
// every unscanned point is at least r h - slack away, so the search stops once the k-th squared distance is below that bound
// squared (with a relative margin of 1e-12 for the rounding of d2), once the bound reaches the radius, or when every cell has
// been scanned.  The query's own point is a candidate like any other.
__global__ void __launch_bounds__(256) nm_knn_kernel(const double* __restrict__ pts, const CloudSeg* __restrict__ segs,
                                                     const NmCloud* __restrict__ clouds, const int* __restrict__ status, int knn,
                                                     double radius, const unsigned long long* __restrict__ tab_key,
                                                     const int* __restrict__ tab_start, const int* __restrict__ tab_cnt,
                                                     const double* __restrict__ sxyz, const int* __restrict__ sidx,
                                                     double* __restrict__ out, int* __restrict__ out_nbr, double* __restrict__ out_cov) {
    if (*status) return;
    const CloudSeg sg = segs[blockIdx.y];
    const int lane = threadIdx.x & 31;
    const int qs = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (qs >= sg.len) return;
    const NmCloud c = clouds[blockIdx.y];
    const long long qrow = sg.start + qs;
    const double qx = sxyz[3 * qrow], qy = sxyz[3 * qrow + 1], qz = sxyz[3 * qrow + 2];
    const int qi = sidx[qrow];
    const int cx = cell_of(qx, c.lo[0], c.h), cy = cell_of(qy, c.lo[1], c.h), cz = cell_of(qz, c.lo[2], c.h);
    const bool hybrid = radius > 0.0;
    const double r2 = dm(radius, radius);
    const unsigned tsize = 2u * (unsigned)sg.len;
    const long long tbase = 2ll * sg.start;

    double d_lo = INFINITY, d_hi = INFINITY;     // top-k entries lane and lane + 32
    int i_lo = 0x7fffffff, i_hi = 0x7fffffff;
    int filled = 0;                              // entries held, <= knn
    int seen = 0;                                // points of the scanned cells
    double kth_d = INFINITY;                     // entry knn - 1 (infinite until knn are held)
    int kth_i = 0x7fffffff;
    const int kl = (knn - 1) & 31;
    const bool kh = (knn - 1) >= 32;

    for (int r = 0;; ++r) {
        const int z0 = max(cz - r, 0), z1 = min(cz + r, c.dims[2] - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, c.dims[1] - 1);
        const int x0 = max(cx - r, 0), x1 = min(cx + r, c.dims[0] - 1);
        auto visit = [&](int x, int y, int z) {
            // the cell's run in the cell order
            const unsigned long long key = pack_cell(x, y, z);
            unsigned h = (unsigned)(mix64(key) % tsize);
            int start = 0, cnt = 0;
            while (true) {
                const unsigned long long k = tab_key[tbase + h];
                if (k == key) { start = tab_start[tbase + h]; cnt = tab_cnt[tbase + h]; break; }
                if (k == kEmpty) break;
                h = (h + 1 == tsize) ? 0 : h + 1;
            }
            for (int j0 = 0; j0 < cnt; j0 += 32) {
                const int j = j0 + lane;
                double d2 = INFINITY;
                int ci = 0x7fffffff;
                if (j < cnt) {
                    const long long row = sg.start + start + j;
                    const double dx = ds(qx, sxyz[3 * row]), dy = ds(qy, sxyz[3 * row + 1]), dz = ds(qz, sxyz[3 * row + 2]);
                    d2 = da(da(dm(dx, dx), dm(dy, dy)), dm(dz, dz));
                    ci = sidx[row];
                }
                bool pass = j < cnt && (!hybrid || d2 < r2) && before(d2, ci, kth_d, kth_i);
                unsigned m = __ballot_sync(0xffffffffu, pass);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const double cd = __shfl_sync(0xffffffffu, d2, src);
                    const int cidx = __shfl_sync(0xffffffffu, ci, src);
                    if (!before(cd, cidx, kth_d, kth_i)) continue;     // the list moved on since the ballot
                    const int pos = __popc(__ballot_sync(0xffffffffu, !before(cd, cidx, d_lo, i_lo))) +
                                    __popc(__ballot_sync(0xffffffffu, !before(cd, cidx, d_hi, i_hi)));
                    const double up_lo_d = __shfl_up_sync(0xffffffffu, d_lo, 1);
                    const int up_lo_i = __shfl_up_sync(0xffffffffu, i_lo, 1);
                    const double up_hi_d = __shfl_up_sync(0xffffffffu, d_hi, 1);
                    const int up_hi_i = __shfl_up_sync(0xffffffffu, i_hi, 1);
                    const double last_lo_d = __shfl_sync(0xffffffffu, d_lo, 31);
                    const int last_lo_i = __shfl_sync(0xffffffffu, i_lo, 31);
                    if (lane > pos) { d_lo = up_lo_d; i_lo = up_lo_i; }
                    else if (lane == pos) { d_lo = cd; i_lo = cidx; }
                    const int ph = lane + 32;
                    if (ph > pos) {
                        d_hi = lane == 0 ? last_lo_d : up_hi_d;
                        i_hi = lane == 0 ? last_lo_i : up_hi_i;
                    } else if (ph == pos) { d_hi = cd; i_hi = cidx; }
                    filled = min(filled + 1, knn);
                    if (filled == knn) {
                        kth_d = __shfl_sync(0xffffffffu, kh ? d_hi : d_lo, kl);
                        kth_i = __shfl_sync(0xffffffffu, kh ? i_hi : i_lo, kl);
                    }
                }
            }
            seen += cnt;
        };
        for (int z = z0; z <= z1; ++z) {
            for (int y = y0; y <= y1; ++y) {
                if (abs(z - cz) == r || abs(y - cy) == r) {
                    for (int x = x0; x <= x1; ++x) visit(x, y, z);
                } else {
                    if (cx - r >= 0) visit(cx - r, y, z);
                    if (cx + r < c.dims[0]) visit(cx + r, y, z);
                }
            }
        }
        if (seen == sg.len) break;     // every point of the cloud has been a candidate
        const bool all = cx - r <= 0 && cy - r <= 0 && cz - r <= 0 && cx + r >= c.dims[0] - 1 && cy + r >= c.dims[1] - 1 &&
                         cz + r >= c.dims[2] - 1;
        if (all) break;
        const double bound = ds(dm((double)r, c.h), c.slack);
        if (bound > 0.0) {
            const double b2 = dm(dm(bound, bound), 1.0 - 1e-12);
            if (filled == knn && kth_d < b2) break;
            if (hybrid && b2 >= r2) break;
        }
    }

    // positions 0..filled-1 hold the neighbours in ascending (d2, index); lane j loads neighbours j and j + 32
    const long long base = 3ll * sg.start;
    double px_lo = 0.0, py_lo = 0.0, pz_lo = 0.0, px_hi = 0.0, py_hi = 0.0, pz_hi = 0.0;
    if (lane < filled) { px_lo = pts[base + 3ll * i_lo]; py_lo = pts[base + 3ll * i_lo + 1]; pz_lo = pts[base + 3ll * i_lo + 2]; }
    if (lane + 32 < filled) { px_hi = pts[base + 3ll * i_hi]; py_hi = pts[base + 3ll * i_hi + 1]; pz_hi = pts[base + 3ll * i_hi + 2]; }
    double cum[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int t = 0; t < filled; ++t) {
        const bool hi = t >= 32;
        const double x = __shfl_sync(0xffffffffu, hi ? px_hi : px_lo, t & 31);
        const double y = __shfl_sync(0xffffffffu, hi ? py_hi : py_lo, t & 31);
        const double z = __shfl_sync(0xffffffffu, hi ? pz_hi : pz_lo, t & 31);
        cum[0] = da(cum[0], x);
        cum[1] = da(cum[1], y);
        cum[2] = da(cum[2], z);
        cum[3] = da(cum[3], dm(x, x));
        cum[4] = da(cum[4], dm(x, y));
        cum[5] = da(cum[5], dm(x, z));
        cum[6] = da(cum[6], dm(y, y));
        cum[7] = da(cum[7], dm(y, z));
        cum[8] = da(cum[8], dm(z, z));
    }
    const long long orow = sg.start + qi;
    if (out_nbr != nullptr) {
        if (lane < knn) out_nbr[orow * knn + lane] = lane < filled ? i_lo : -1;
        if (lane + 32 < knn) out_nbr[orow * knn + lane + 32] = lane + 32 < filled ? i_hi : -1;
    }
    if (lane != 0) return;
    Sym3 A = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (filled > 0) {
        const double cnt = (double)filled;
#pragma unroll
        for (int a = 0; a < 9; ++a) cum[a] = dd(cum[a], cnt);
        A = {ds(cum[3], dm(cum[0], cum[0])), ds(cum[4], dm(cum[0], cum[1])), ds(cum[5], dm(cum[0], cum[2])),
             ds(cum[6], dm(cum[1], cum[1])), ds(cum[7], dm(cum[1], cum[2])), ds(cum[8], dm(cum[2], cum[2]))};
    }
    if (out_cov != nullptr) {
        double* o = out_cov + 6 * orow;
        o[0] = A.a00; o[1] = A.a01; o[2] = A.a02; o[3] = A.a11; o[4] = A.a12; o[5] = A.a22;
    }
    V3 n = {0.0, 0.0, 1.0};
    if (filled >= 3) {
        const V3 e = fast_eigen3x3(A);
        // normal.norm() == 0.0, with Eigen's (x^2 + y^2) + z^2
        if (!(sqrt(da(da(dm(e.x, e.x), dm(e.y, e.y)), dm(e.z, e.z))) == 0.0)) n = e;
    }
    out[3 * orow + 0] = n.x;
    out[3 * orow + 1] = n.y;
    out[3 * orow + 2] = n.z;
}

// numpy's regularize_normals, row by row: d = -(((x nx) + y ny) + z nz) in T (numpy's type of points * normals), dir = d > 0;
// positive: n dir - n (1 - dir), otherwise n (1 - dir) - n dir.  numpy takes n * dir (a bool) in T and n * (1 - dir) (an int64)
// in double, so the difference and the result are double for either T.
template <typename T>
__global__ void nm_regularize_kernel(const T* __restrict__ p, const T* __restrict__ nrm, int64_t n, int positive, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T* a = p + 3 * i;
    const T* b = nrm + 3 * i;
    T s;
    if constexpr (sizeof(T) == 8) s = -__dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
    else s = -__fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
    const bool dir = s > T(0);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double by_bool = (double)(b[k] * T(dir ? 1 : 0));           // n * direction, in T
        const double by_int = __dmul_rn((double)b[k], dir ? 0.0 : 1.0);    // n * (1 - direction), in double
        out[3 * i + k] = positive ? __dsub_rn(by_bool, by_int) : __dsub_rn(by_int, by_bool);
    }
}

}  // namespace

}  // namespace geob200

using namespace geob200;

extern "C" {

size_t geob200_estimate_normals_workspace_bytes(int64_t n_points, int64_t batch) {
    if (n_points < 0 || batch < 0) return 0;
    const size_t n = (size_t)n_points, b = (size_t)batch;
    size_t bytes = align_up(sizeof(CloudSeg) * 2 * b, 256) + align_up(sizeof(NmCloud) * b, 256);
    bytes += align_up(8 * 2 * n, 256) + align_up(4 * 2 * n, 256) * 3;   // tab_key, tab_cnt, tab_start, tab_fill
    bytes += align_up(4 * n, 256) * 2;                                  // pt_slot, sorted_idx
    bytes += align_up(8 * 3 * n, 256);                                  // sorted_xyz
    bytes += 256;                                                       // status
    return bytes + 4096;
}

int geob200_estimate_normals(const double* points, int64_t n_points, const int64_t* lengths_h, int64_t batch, int64_t knn, double radius,
                             double* out_normals, int32_t* out_neighbors, double* out_covariance, int64_t* out_status, void* workspace,
                             size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GEOB_REQUIRE(batch >= 1 && batch <= GEOB200_NORMALS_MAX_CLOUDS, "estimate_normals: batch must be in 1..%d, got %lld",
                 GEOB200_NORMALS_MAX_CLOUDS, (long long)batch);
    GEOB_REQUIRE(lengths_h != nullptr && out_status != nullptr, "estimate_normals: null lengths or status pointer");
    GEOB_REQUIRE(n_points >= 0 && n_points < (1ll << 30), "estimate_normals: n_points must be in 0..2^30-1, got %lld",
                 (long long)n_points);
    GEOB_REQUIRE(knn >= 1 && knn <= GEOB200_NORMALS_MAX_KNN, "estimate_normals: knn must be in 1..%d, got %lld", GEOB200_NORMALS_MAX_KNN,
                 (long long)knn);
    GEOB_REQUIRE(radius == 0.0 || (radius > 0.0 && isfinite(radius)), "estimate_normals: radius must be 0 (none) or positive and finite, got %g",
                 radius);
    int64_t total = 0;
    int max_len = 0;
    for (int64_t b = 0; b < batch; ++b) {
        GEOB_REQUIRE(lengths_h[b] >= 0, "estimate_normals: cloud %lld has a negative length", (long long)b);
        total += lengths_h[b];
        if (lengths_h[b] > max_len) max_len = (int)lengths_h[b];
    }
    GEOB_REQUIRE(total == n_points, "estimate_normals: sum(lengths)=%lld != n_points=%lld", (long long)total, (long long)n_points);
    GEOB_REQUIRE(n_points == 0 || (points != nullptr && out_normals != nullptr), "estimate_normals: null point pointer");
    GEOB_REQUIRE(workspace != nullptr && workspace_bytes >= geob200_estimate_normals_workspace_bytes(n_points, batch),
                 "estimate_normals: workspace too small (%zu bytes, need %zu)", workspace_bytes,
                 geob200_estimate_normals_workspace_bytes(n_points, batch));

    Arena ar(workspace, workspace_bytes);
    const size_t n = (size_t)n_points;
    CloudSeg* segs = ar.take<CloudSeg>(2 * batch);   // the clouds' rows, then their table slots
    CloudSeg* tsegs = segs + batch;
    NmCloud* clouds = ar.take<NmCloud>(batch);
    unsigned long long* tab_key = ar.take<unsigned long long>(2 * n);
    int* tab_cnt = ar.take<int>(2 * n);
    int* tab_start = ar.take<int>(2 * n);
    int* tab_fill = ar.take<int>(2 * n);
    int* pt_slot = ar.take<int>(n);
    int* sorted_idx = ar.take<int>(n);
    double* sorted_xyz = ar.take<double>(3 * n);
    int* status = ar.take<int>(64);
    GEOB_REQUIRE(ar.ok(), "estimate_normals: workspace accounting error");

    CloudSeg h[2 * GEOB200_NORMALS_MAX_CLOUDS];
    for (int64_t b = 0, acc = 0; b < batch; acc += lengths_h[b], ++b) {
        h[b].start = (int)acc;
        h[b].len = (int)lengths_h[b];
        h[batch + b].start = 2 * (int)acc;     // the cloud's table slots
        h[batch + b].len = 2 * (int)lengths_h[b];
    }
    GEOB_CHECK_CUDA(cudaMemcpyAsync(segs, h, sizeof(CloudSeg) * 2 * batch, cudaMemcpyHostToDevice, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
    if (n == 0) {
        GEOB_CHECK_CUDA(cudaMemsetAsync(out_status, 0, sizeof(int64_t), st));
        return 0;
    }
    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_key, 0xFF, 8 * 2 * n, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_cnt, 0, 4 * 2 * n, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync(tab_fill, 0, 4 * 2 * n, st));

    const unsigned nbt = (unsigned)batch;
    const dim3 pgrid((max_len + 255) / 256, nbt);
    nm_bounds_kernel<<<nbt, 1024, 0, st>>>(points, segs, (int)knn, radius, clouds, status);
    nm_insert_kernel<<<pgrid, 256, 0, st>>>(points, segs, clouds, status, tab_key, tab_cnt, pt_slot);
    seg_exclusive_scan_kernel<<<nbt, 1024, 0, st>>>(tab_cnt, tab_start, tsegs, nullptr);
    nm_scatter_kernel<<<pgrid, 256, 0, st>>>(points, segs, status, pt_slot, tab_start, tab_fill, sorted_xyz, sorted_idx);
    const dim3 qgrid((max_len + 7) / 8, nbt);
    nm_knn_kernel<<<qgrid, 256, 0, st>>>(points, segs, clouds, status, (int)knn, radius, tab_key, tab_start, tab_cnt, sorted_xyz,
                                         sorted_idx, out_normals, out_neighbors, out_covariance);
    GEOB_CHECK_CUDA(cudaMemcpyAsync(out_status, status, sizeof(int), cudaMemcpyDeviceToDevice, st));
    GEOB_CHECK_CUDA(cudaMemsetAsync((char*)out_status + 4, 0, 4, st));
    GEOB_CHECK_LAUNCH();
    count_launches(5);
    return 0;
}

int geob200_regularize_normals(const void* points, const void* normals, int64_t n, int fp64, int positive, double* out, void* stream) {
    GEOB_REQUIRE(n >= 0, "regularize_normals: negative row count %lld", (long long)n);
    GEOB_REQUIRE(n == 0 || (points != nullptr && normals != nullptr && out != nullptr), "regularize_normals: null pointer");
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (fp64) nm_regularize_kernel<double><<<grid, 256, 0, st>>>((const double*)points, (const double*)normals, n, positive, (double*)out);
    else nm_regularize_kernel<float><<<grid, 256, 0, st>>>((const float*)points, (const float*)normals, n, positive, (double*)out);
    GEOB_CHECK_LAUNCH();
    count_launches(1);
    return 0;
}

}  // extern "C"
