// TEST INFRASTRUCTURE ONLY.  A plain C++ restatement of Open3D's PointCloud::EstimateNormals with FastEigen3x3 (Open3D 0.11.2,
// no prior normals, so no orientation), the contract that geob200_estimate_normals (geotransformer_b200/csrc/normals.cu)
// implements on the device:
//
//   p_i in double (float32 inputs are widened exactly); d2(i, j) = ((dx dx) + dy dy) + dz dz, dx = p_i.x - p_j.x, no FMA;
//   neighbours of p_i: all points in ascending (d2, index), with a radius only those with d2 < radius * radius, cut to knn;
//   cumulants x, y, z, xx, xy, xz, yy, yz, zz added over the neighbours in that order from 0, each divided by double(count);
//   covariance entry ab = E[ab] - E[a] E[b];
//   normal: FastEigen3x3 of the covariance; (0, 0, 1) when there are fewer than 3 neighbours or the result's norm is 0.
//
// The neighbours come from a brute-force full sort by (d2, index), so the oracle shares no search code with the device.
// Parity with Open3D itself is not verified here: Open3D is not a dependency of this project.
// Built without -ffast-math and without -march=native (x86-64 baseline has no FMA).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <numeric>
#include <vector>

namespace {

struct V3 {
    double x, y, z;
};

V3 cross(const V3& a, const V3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
// Eigen 3.3's dot of two 3-vectors: one packet of two doubles, then the third product
double dot(const V3& a, const V3& b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
V3 div(const V3& a, double s) { return {a.x / s, a.y / s, a.z / s}; }

struct Sym3 {
    double a00, a01, a02, a11, a12, a22;
};

V3 eigenvector0(const Sym3& A, double ev) {
    const V3 r0 = {A.a00 - ev, A.a01, A.a02}, r1 = {A.a01, A.a11 - ev, A.a12}, r2 = {A.a02, A.a12, A.a22 - ev};
    const V3 r0xr1 = cross(r0, r1), r0xr2 = cross(r0, r2), r1xr2 = cross(r1, r2);
    const double d0 = dot(r0xr1, r0xr1), d1 = dot(r0xr2, r0xr2), d2 = dot(r1xr2, r1xr2);
    double dmax = d0;
    int imax = 0;
    if (d1 > dmax) {
        dmax = d1;
        imax = 1;
    }
    if (d2 > dmax) imax = 2;
    if (imax == 0) return div(r0xr1, std::sqrt(d0));
    if (imax == 1) return div(r0xr2, std::sqrt(d1));
    return div(r1xr2, std::sqrt(d2));
}

V3 eigenvector1(const Sym3& A, const V3& e0, double ev) {
    V3 U;
    if (std::abs(e0.x) > std::abs(e0.y)) {
        const double inv = 1 / std::sqrt(e0.x * e0.x + e0.z * e0.z);
        U = {-e0.z * inv, 0, e0.x * inv};
    } else {
        const double inv = 1 / std::sqrt(e0.y * e0.y + e0.z * e0.z);
        U = {0, e0.z * inv, -e0.y * inv};
    }
    const V3 V = cross(e0, U);
    const V3 AU = {A.a00 * U.x + A.a01 * U.y + A.a02 * U.z, A.a01 * U.x + A.a11 * U.y + A.a12 * U.z,
                   A.a02 * U.x + A.a12 * U.y + A.a22 * U.z};
    const V3 AV = {A.a00 * V.x + A.a01 * V.y + A.a02 * V.z, A.a01 * V.x + A.a11 * V.y + A.a12 * V.z,
                   A.a02 * V.x + A.a12 * V.y + A.a22 * V.z};
    double m00 = U.x * AU.x + U.y * AU.y + U.z * AU.z - ev;
    double m01 = U.x * AV.x + U.y * AV.y + U.z * AV.z;
    double m11 = V.x * AV.x + V.y * AV.y + V.z * AV.z - ev;
    const double abs00 = std::abs(m00), abs01 = std::abs(m01), abs11 = std::abs(m11);
    if (abs00 >= abs11) {
        if (std::max(abs00, abs01) > 0) {
            if (abs00 >= abs01) {
                m01 /= m00;
                m00 = 1 / std::sqrt(1 + m01 * m01);
                m01 *= m00;
            } else {
                m00 /= m01;
                m01 = 1 / std::sqrt(1 + m00 * m00);
                m00 *= m01;
            }
            return {m01 * U.x - m00 * V.x, m01 * U.y - m00 * V.y, m01 * U.z - m00 * V.z};
        }
        return U;
    }
    if (std::max(abs11, abs01) > 0) {
        if (abs11 >= abs01) {
            m01 /= m11;
            m11 = 1 / std::sqrt(1 + m01 * m01);
            m01 *= m11;
        } else {
            m11 /= m01;
            m01 = 1 / std::sqrt(1 + m11 * m11);
            m11 *= m01;
        }
        return {m11 * U.x - m01 * V.x, m11 * U.y - m01 * V.y, m11 * U.z - m01 * V.z};
    }
    return U;
}

V3 fast_eigen3x3(const Sym3& in) {
    const double maxc = std::max({in.a00, in.a01, in.a02, in.a11, in.a12, in.a22});
    if (maxc == 0) return {0, 0, 0};
    const Sym3 A = {in.a00 / maxc, in.a01 / maxc, in.a02 / maxc, in.a11 / maxc, in.a12 / maxc, in.a22 / maxc};
    const double norm = A.a01 * A.a01 + A.a02 * A.a02 + A.a12 * A.a12;
    if (norm > 0) {
        const double q = (A.a00 + A.a11 + A.a22) / 3;
        const double b00 = A.a00 - q, b11 = A.a11 - q, b22 = A.a22 - q;
        const double p = std::sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6);
        const double c00 = b11 * b22 - A.a12 * A.a12;
        const double c01 = A.a01 * b22 - A.a12 * A.a02;
        const double c02 = A.a01 * A.a12 - b11 * A.a02;
        const double det = (b00 * c00 - A.a01 * c01 + A.a02 * c02) / (p * p * p);
        const double half_det = std::min(std::max(det * 0.5, -1.0), 1.0);
        const double angle = std::acos(half_det) / (double)3;
        const double two_thirds_pi = 2.09439510239319549;
        const double beta2 = std::cos(angle) * 2;
        const double beta0 = std::cos(angle + two_thirds_pi) * 2;
        const double beta1 = -(beta0 + beta2);
        const double ev0 = q + p * beta0, ev1 = q + p * beta1, ev2 = q + p * beta2;
        if (half_det >= 0) {
            const V3 e2 = eigenvector0(A, ev2);
            if (ev2 < ev0 && ev2 < ev1) return e2;
            const V3 e1 = eigenvector1(A, e2, ev1);
            if (ev1 < ev0 && ev1 < ev2) return e1;
            return cross(e1, e2);
        }
        const V3 e0 = eigenvector0(A, ev0);
        if (ev0 < ev1 && ev0 < ev2) return e0;
        const V3 e1 = eigenvector1(A, e0, ev1);
        if (ev1 < ev0 && ev1 < ev2) return e1;
        return cross(e0, e1);
    }
    // A *= maxc restores the matrix before Open3D compares the diagonal entries
    const double d0 = A.a00 * maxc, d1 = A.a11 * maxc, d2 = A.a22 * maxc;
    if (d0 < d1 && d0 < d2) return {1, 0, 0};
    if (d1 < d0 && d1 < d2) return {0, 1, 0};
    return {0, 0, 1};
}

}  // namespace

extern "C" {

enum { NRM_OK = 0, NRM_NONFINITE = 1, NRM_BAD_ARG = 2 };

// One cloud; the queries are the points rows[0..n_rows) (rows == NULL: every point, n_rows ignored).  Row r of the outputs
// belongs to query r.  out_normals: 3 per query; out_neighbors (optional): knn in-cloud indices per query, -1 past the count;
// out_cov (optional): 6 per query (c00 c01 c02 c11 c12 c22).  radius <= 0: no radius.  Returns 0 or an error code (nothing is
// written then).
int normals_oracle(const double* points, int64_t n, int64_t knn, double radius, const int64_t* rows, int64_t n_rows,
                   double* out_normals, int32_t* out_neighbors, double* out_cov) {
    if (knn < 1) return NRM_BAD_ARG;
    for (int64_t i = 0; i < 3 * n; ++i)
        if (!std::isfinite(points[i])) return NRM_NONFINITE;
    const bool hybrid = radius > 0;
    const double r2 = radius * radius;
    std::vector<double> d2((size_t)n);
    std::vector<int32_t> order((size_t)n);
    if (rows == nullptr) n_rows = n;
    for (int64_t r = 0; r < n_rows; ++r)
        if (rows != nullptr && (rows[r] < 0 || rows[r] >= n)) return NRM_BAD_ARG;
    for (int64_t i = 0; i < n_rows; ++i) {
        const double* q = points + 3 * (rows == nullptr ? i : rows[i]);
        for (int64_t j = 0; j < n; ++j) {
            const double* p = points + 3 * j;
            const double dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
            d2[j] = dx * dx + dy * dy + dz * dz;
        }
        std::iota(order.begin(), order.end(), 0);
        std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return d2[a] < d2[b] || (d2[a] == d2[b] && a < b); });
        int64_t cnt = std::min<int64_t>(knn, n);
        if (hybrid) {
            int64_t m = 0;
            while (m < cnt && d2[order[m]] < r2) ++m;
            cnt = m;
        }
        if (out_neighbors != nullptr)
            for (int64_t t = 0; t < knn; ++t) out_neighbors[i * knn + t] = t < cnt ? order[t] : -1;
        double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int64_t t = 0; t < cnt; ++t) {
            const double* p = points + 3 * order[t];
            c[0] += p[0];
            c[1] += p[1];
            c[2] += p[2];
            c[3] += p[0] * p[0];
            c[4] += p[0] * p[1];
            c[5] += p[0] * p[2];
            c[6] += p[1] * p[1];
            c[7] += p[1] * p[2];
            c[8] += p[2] * p[2];
        }
        Sym3 A = {0, 0, 0, 0, 0, 0};
        if (cnt > 0) {
            for (double& v : c) v /= (double)cnt;
            A = {c[3] - c[0] * c[0], c[4] - c[0] * c[1], c[5] - c[0] * c[2], c[6] - c[1] * c[1], c[7] - c[1] * c[2], c[8] - c[2] * c[2]};
        }
        if (out_cov != nullptr) {
            double* o = out_cov + 6 * i;
            o[0] = A.a00; o[1] = A.a01; o[2] = A.a02; o[3] = A.a11; o[4] = A.a12; o[5] = A.a22;
        }
        V3 nrm = {0, 0, 1};
        if (cnt >= 3) {
            const V3 e = fast_eigen3x3(A);
            if (!(std::sqrt((e.x * e.x + e.y * e.y) + e.z * e.z) == 0.0)) nrm = e;
        }
        out_normals[3 * i] = nrm.x;
        out_normals[3 * i + 1] = nrm.y;
        out_normals[3 * i + 2] = nrm.z;
    }
    return NRM_OK;
}

// FastEigen3x3 of one covariance (c00 c01 c02 c11 c12 c22), for tests of the eigensolver's branches
void normals_oracle_eigen(const double* cov, double* out) {
    const V3 e = fast_eigen3x3({cov[0], cov[1], cov[2], cov[3], cov[4], cov[5]});
    out[0] = e.x;
    out[1] = e.y;
    out[2] = e.z;
}

}  // extern "C"
