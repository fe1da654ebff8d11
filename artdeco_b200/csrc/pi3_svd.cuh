// 3x3 SVD orthogonalisation of Pi3's camera head (VSLAM/thirdparty/Pi3/pi3/models/layers/camera_head.py:74-93), in fp64:
//   A = normalize_rows(m)^T = U S V^T,  R = V diag(1, 1, det(V U^T)) U^T.
// One-sided (Hestenes) Jacobi on the columns of A accumulates V; the column norms are S and the normalised columns U.
// R is independent of the SVD's sign choices: flipping a (u_i, v_i) pair leaves v_i u_i^T unchanged, and flipping u_3
// or v_3 alone also flips det(V U^T).  So u_3 is always taken as u_1 x u_2, which also completes U when A is rank 2;
// when A is rank 1, u_2 is any unit vector orthogonal to u_1 (R is then not unique, but it is still a rotation).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define ADB_HD __host__ __device__ __forceinline__
#else
#define ADB_HD inline
#endif

ADB_HD void adb_pi3_svd_orthogonalize(const double m[9], double R[9]) {
    double A[3][3], V[3][3];
    for (int r = 0; r < 3; ++r) {
        const double n = sqrt(m[r * 3] * m[r * 3] + m[r * 3 + 1] * m[r * 3 + 1] + m[r * 3 + 2] * m[r * 3 + 2]);
        const double inv = 1.0 / (n > 1e-12 ? n : 1e-12);           // F.normalize(p=2, eps=1e-12)
        for (int c = 0; c < 3; ++c) A[c][r] = m[r * 3 + c] * inv;   // transpose
    }
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) V[r][c] = r == c ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 32; ++sweep) {
        bool rotated = false;
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            double al = 0, be = 0, ga = 0;
            for (int i = 0; i < 3; ++i) { al += A[i][p] * A[i][p]; be += A[i][q] * A[i][q]; ga += A[i][p] * A[i][q]; }
            if (ga == 0.0 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
            rotated = true;
            const double zeta = (be - al) / (2.0 * ga);
            const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
            for (int i = 0; i < 3; ++i) {
                const double ap = A[i][p], aq = A[i][q];
                A[i][p] = c * ap - s * aq; A[i][q] = s * ap + c * aq;
                const double vp = V[i][p], vq = V[i][q];
                V[i][p] = c * vp - s * vq; V[i][q] = s * vp + c * vq;
            }
        }
        if (!rotated) break;
    }
    double sv[3];
    int ord[3] = {0, 1, 2};
    for (int j = 0; j < 3; ++j) sv[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
    for (int a = 0; a < 2; ++a)                     // descending singular values
        for (int b = 0; b < 2 - a; ++b)
            if (sv[ord[b]] < sv[ord[b + 1]]) { const int t = ord[b]; ord[b] = ord[b + 1]; ord[b + 1] = t; }
    double u[3][3], v[3][3];                        // u[k], v[k]: k-th singular vectors
    for (int k = 0; k < 3; ++k)
        for (int i = 0; i < 3; ++i) v[k][i] = V[i][ord[k]];
    const double s0 = sv[ord[0]];
    for (int i = 0; i < 3; ++i) u[0][i] = s0 > 0 ? A[i][ord[0]] / s0 : (i == 0 ? 1.0 : 0.0);
    {
        double w[3], d = 0;
        for (int i = 0; i < 3; ++i) w[i] = A[i][ord[1]];
        for (int i = 0; i < 3; ++i) d += u[0][i] * w[i];
        for (int i = 0; i < 3; ++i) w[i] -= d * u[0][i];
        double n = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
        if (!(n > 1e-12 * (s0 > 0 ? s0 : 1.0))) {  // rank 1: any unit vector orthogonal to u_0
            const int ax = (fabs(u[0][0]) <= fabs(u[0][1]) && fabs(u[0][0]) <= fabs(u[0][2])) ? 0 : (fabs(u[0][1]) <= fabs(u[0][2]) ? 1 : 2);
            double e[3] = {0, 0, 0};
            e[ax] = 1.0;
            w[0] = u[0][1] * e[2] - u[0][2] * e[1];
            w[1] = u[0][2] * e[0] - u[0][0] * e[2];
            w[2] = u[0][0] * e[1] - u[0][1] * e[0];
            n = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
        }
        for (int i = 0; i < 3; ++i) u[1][i] = w[i] / n;
    }
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    // det(U) = +1 by construction, so det(V U^T) = det(V)
    const double dv = v[0][0] * (v[1][1] * v[2][2] - v[1][2] * v[2][1]) - v[0][1] * (v[1][0] * v[2][2] - v[1][2] * v[2][0]) +
                      v[0][2] * (v[1][0] * v[2][1] - v[1][1] * v[2][0]);
    const double d = dv < 0 ? -1.0 : 1.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[r * 3 + c] = v[0][r] * u[0][c] + v[1][r] * u[1][c] + d * v[2][r] * u[2][c];
}
