// 3x3 SVD / Kabsch rotation in double, shared by LGR (lgr.cu) and correspondence RANSAC (ransac.cu).
#pragma once

namespace geob200 {

// One-sided Jacobi: H V = U S.  Returns R = V diag(1,1,sign(det(V U^T))) U^T  (procrustes.py:53-57).
__device__ inline void kabsch_rotation(const double Hin[9], double R[9]) {
    double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double fro = 0.0;
    for (int i = 0; i < 9; ++i) { A[i] = Hin[i]; fro += Hin[i] * Hin[i]; }
    if (!(fro > 0.0)) {                       // H == 0: LAPACK returns U = V = I  ->  R = I
        for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
        return;
    }
    for (int sweep = 0; sweep < 40; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double al = 0, be = 0, ga = 0;
                for (int i = 0; i < 3; ++i) { al += A[3 * i + p] * A[3 * i + p]; be += A[3 * i + q] * A[3 * i + q]; ga += A[3 * i + p] * A[3 * i + q]; }
                off += ga * ga;
                if (fabs(ga) <= 1e-300 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
                const double zeta = (be - al) / (2.0 * ga);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int i = 0; i < 3; ++i) {
                    const double ap = A[3 * i + p], aq = A[3 * i + q];
                    A[3 * i + p] = c * ap - s * aq; A[3 * i + q] = s * ap + c * aq;
                    const double vp = V[3 * i + p], vq = V[3 * i + q];
                    V[3 * i + p] = c * vp - s * vq; V[3 * i + q] = s * vp + c * vq;
                }
            }
        if (off <= 1e-34 * fro * fro) break;
    }
    double sv[3];
    for (int j = 0; j < 3; ++j) sv[j] = sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
    int ord[3] = {0, 1, 2};                   // descending singular values (LAPACK order: flip applies to the smallest)
    for (int a = 0; a < 2; ++a)
        for (int b = a + 1; b < 3; ++b)
            if (sv[ord[b]] > sv[ord[a]]) { int t = ord[a]; ord[a] = ord[b]; ord[b] = t; }
    double U[9], Vs[9];
    for (int j = 0; j < 3; ++j) {
        const int o = ord[j];
        for (int i = 0; i < 3; ++i) { Vs[3 * i + j] = V[3 * i + o]; U[3 * i + j] = A[3 * i + o]; }
    }
    const double tol = 1e-14 * sv[ord[0]];
    for (int j = 0; j < 3; ++j) {
        const double s = sv[ord[j]];
        if (s > tol) { for (int i = 0; i < 3; ++i) U[3 * i + j] /= s; }
        else {
            // rank-deficient: complete U to an orthonormal basis
            double c[3];
            if (j == 2) {
                c[0] = U[3] * U[7] - U[6] * U[4]; c[1] = U[6] * U[1] - U[0] * U[7]; c[2] = U[0] * U[4] - U[3] * U[1];
            } else {  // j == 1 (rank 1): any unit vector orthogonal to column 0
                const double a0 = fabs(U[0]), a1 = fabs(U[3]), a2 = fabs(U[6]);
                double e[3] = {0, 0, 0};
                e[(a0 <= a1 && a0 <= a2) ? 0 : (a1 <= a2 ? 1 : 2)] = 1.0;
                const double d = e[0] * U[0] + e[1] * U[3] + e[2] * U[6];
                c[0] = e[0] - d * U[0]; c[1] = e[1] - d * U[3]; c[2] = e[2] - d * U[6];
            }
            const double n = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
            for (int i = 0; i < 3; ++i) U[3 * i + j] = c[i] / n;
        }
    }
    // M = V U^T ; det ; R = V diag(1,1,sign) U^T
    double M[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M[3 * i + j] = Vs[3 * i] * U[3 * j] + Vs[3 * i + 1] * U[3 * j + 1] + Vs[3 * i + 2] * U[3 * j + 2];
    const double det = M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
    const double sg = det > 0 ? 1.0 : (det < 0 ? -1.0 : 0.0);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[3 * i + j] = Vs[3 * i] * U[3 * j] + Vs[3 * i + 1] * U[3 * j + 1] + sg * Vs[3 * i + 2] * U[3 * j + 2];
}

}  // namespace geob200
