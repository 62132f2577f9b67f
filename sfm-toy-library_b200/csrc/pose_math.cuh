// pose_math.cuh -- per-sample arithmetic of the PnP RANSAC (pose.cu): the EPnP minimal solver on five 2D-3D correspondences and
// the rotation-matrix -> angle-axis conversion the refit starts from.
//
// EPnP (Lepetit, Moreno-Noguer, Fua, "EPnP: An Accurate O(n) Solution to the PnP Problem", IJCV 2009), the algorithm of
// cv::solvePnP(SOLVEPNP_EPNP), which cv::solvePnPRansac runs on its minimal sets, in fp64:
//   1. control points: c0 the centroid of the world points, c1..c3 = c0 + sqrt(lambda_j / n) e_j along the principal axes
//      (eigen-decomposition of the 3 x 3 scatter matrix by cyclic Jacobi, eigenvalues descending);
//   2. barycentric coordinates alpha of every point in that frame;
//   3. M (2n x 12) from alpha, K and the pixels; M^T M and its 4 smallest eigenvectors by cyclic Jacobi;
//   4. the betas of OpenCV's three initialisations (4, 2 and 3 unknowns, least squares on the 6 x 10 system L beta = rho), each
//      polished by 5 Gauss-Newton steps;
//   5. per initialisation the camera-frame control points, their sign fixed so that the first point lies in front, and R, t by
//      Procrustes (3 x 3 one-sided Jacobi SVD; a reflection flips the last row of R, as OpenCV does);
//   6. the solution with the lowest mean reprojection error on the sample, as epnp::compute_pose keeps.
// A degenerate sample -- coincident, collinear or coplanar world points, a rank-deficient system, a non-finite result -- gives no
// pose (pm_epnp returns false); every returned entry is finite.
// __host__ __device__, so tests compile the very same code with g++ and compare it with cv2.solvePnP(SOLVEPNP_EPNP).
#pragma once
#include <cfloat>
#include <cmath>

#if defined(__CUDACC__)
#define PM_HD __host__ __device__ __forceinline__
#else
#define PM_HD inline
#endif

constexpr int PM_N = 5;    // correspondences of a minimal sample

// Cyclic Jacobi eigen-decomposition of the symmetric N x N matrix A (row-major, destroyed: its diagonal ends up holding the
// eigenvalues), eigenvectors in the columns of V.  The routine of hm_jacobi_min9 (homography_math.cuh) for any N.
template <int N>
PM_HD void pm_jacobi(double* A, double* V) {
    for (int i = 0; i < N * N; ++i) V[i] = (i % (N + 1) == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q) {
                const double apq = A[N * p + q];
                if (apq == 0.0) continue;
                const double app = A[N * p + p], aqq = A[N * q + q], g = 100.0 * fabs(apq);
                if (fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) { A[N * p + q] = A[N * q + p] = 0.0; continue; }
                rotated = true;
                const double theta = (aqq - app) / (2.0 * apq);
                const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < N; ++k) {
                    const double akp = A[N * k + p], akq = A[N * k + q];
                    A[N * k + p] = c * akp - s * akq; A[N * k + q] = s * akp + c * akq;
                }
                for (int k = 0; k < N; ++k) {
                    const double apk = A[N * p + k], aqk = A[N * q + k];
                    A[N * p + k] = c * apk - s * aqk; A[N * q + k] = s * apk + c * aqk;
                }
                A[N * p + q] = A[N * q + p] = 0.0;
                for (int k = 0; k < N; ++k) {
                    const double vkp = V[N * k + p], vkq = V[N * k + q];
                    V[N * k + p] = c * vkp - s * vkq; V[N * k + q] = s * vkp + c * vkq;
                }
            }
        if (!rotated) break;
    }
}

// finite, without isfinite (a macro or a std:: function depending on the compiler)
PM_HD bool pm_finite(double v) { return v - v == 0.0; }

// Least squares min |A x - b| of a 6 x C system (C <= 5) by Householder QR; false when A is rank-deficient.
template <int C>
PM_HD bool pm_lsq6(const double* Ain, const double* bin, double* x) {
    double A[6][C], b[6];
    for (int r = 0; r < 6; ++r) { b[r] = bin[r]; for (int c = 0; c < C; ++c) A[r][c] = Ain[C * r + c]; }
    double amax = 0.0;
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < C; ++c) amax = fmax(amax, fabs(A[r][c]));
    if (!(amax > 0.0) || !(amax < 1e300)) return false;
    double diag[C];
    for (int k = 0; k < C; ++k) {
        double nrm = 0.0;
        for (int r = k; r < 6; ++r) nrm += A[r][k] * A[r][k];
        nrm = sqrt(nrm);
        if (!(nrm > 1e-13 * amax)) return false;
        const double alpha = A[k][k] > 0.0 ? -nrm : nrm;
        double v[6];
        for (int r = k; r < 6; ++r) v[r] = A[r][k];
        v[k] -= alpha;
        double vv = 0.0;
        for (int r = k; r < 6; ++r) vv += v[r] * v[r];
        if (!(vv > 0.0)) return false;
        const double ib = 2.0 / vv;
        for (int c = k + 1; c < C; ++c) {
            double s = 0.0;
            for (int r = k; r < 6; ++r) s += v[r] * A[r][c];
            s *= ib;
            for (int r = k; r < 6; ++r) A[r][c] -= s * v[r];
        }
        double s = 0.0;
        for (int r = k; r < 6; ++r) s += v[r] * b[r];
        s *= ib;
        for (int r = k; r < 6; ++r) b[r] -= s * v[r];
        diag[k] = alpha;
    }
    for (int k = C - 1; k >= 0; --k) {
        double s = b[k];
        for (int c = k + 1; c < C; ++c) s -= A[k][c] * x[c];
        x[k] = s / diag[k];
    }
    for (int k = 0; k < C; ++k)
        if (!pm_finite(x[k])) return false;
    return true;
}

PM_HD double pm_dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// R = U V^T of the 3 x 3 matrix A = U D V^T by one-sided Jacobi (Hestenes) on the columns of A; a reflection (det R < 0) flips
// the last row of R, as epnp::estimate_R_and_t does.  False when A has rank < 2.
PM_HD bool pm_procrustes(const double A[3][3], double R[3][3]) {
    double W[3][3], V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) W[i][j] = A[i][j];
    for (int sweep = 0; sweep < 60; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double al = 0.0, be = 0.0, ga = 0.0;
                for (int k = 0; k < 3; ++k) { al += W[k][p] * W[k][p]; be += W[k][q] * W[k][q]; ga += W[k][p] * W[k][q]; }
                if (!(fabs(ga) > 1e-15 * sqrt(al * be))) continue;
                rotated = true;
                const double zeta = (be - al) / (2.0 * ga);
                const double t = fabs(zeta) > 1e150 ? 0.5 / zeta : (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(zeta * zeta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {
                    const double wp = W[k][p], wq = W[k][q];
                    W[k][p] = c * wp - s * wq; W[k][q] = s * wp + c * wq;
                    const double vp = V[k][p], vq = V[k][q];
                    V[k][p] = c * vp - s * vq; V[k][q] = s * vp + c * vq;
                }
            }
        if (!rotated) break;
    }
    double sg[3];
    for (int j = 0; j < 3; ++j) sg[j] = sqrt(W[0][j] * W[0][j] + W[1][j] * W[1][j] + W[2][j] * W[2][j]);
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2 - i; ++j)
            if (sg[o[j]] < sg[o[j + 1]]) { const int tmp = o[j]; o[j] = o[j + 1]; o[j + 1] = tmp; }
    if (!(sg[o[0]] > 0.0) || !(sg[o[1]] > 1e-12 * sg[o[0]])) return false;
    double U[3][3];    // columns in descending order of the singular values
    for (int j = 0; j < 2; ++j)
        for (int k = 0; k < 3; ++k) U[k][j] = W[k][o[j]] / sg[o[j]];
    if (sg[o[2]] > 1e-12 * sg[o[0]]) {
        for (int k = 0; k < 3; ++k) U[k][2] = W[k][o[2]] / sg[o[2]];
    } else {               // rank 2: the third left singular vector completes a right-handed basis
        U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
        U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
        U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = U[i][0] * V[j][o[0]] + U[i][1] * V[j][o[1]] + U[i][2] * V[j][o[2]];
    const double det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] -
                       R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1];
    if (det < 0) { R[2][0] = -R[2][0]; R[2][1] = -R[2][1]; R[2][2] = -R[2][2]; }
    return true;
}

// The EPnP problem of one sample, kept between the three initialisations.
struct PmEpnp {
    double pw[PM_N][3], us[PM_N][2], alpha[PM_N][4], cw[4][3];
    double fu, fv, uc, vc;
    double ut[4][12];      // eigenvectors of M^T M of the 4 smallest eigenvalues, ascending
    double L[6][10], rho[6];
};

// camera-frame control points and points for betas, the sign fix, Procrustes; returns the mean reprojection error on the
// sample (epnp::reprojection_error), or +inf when the solution is unusable
PM_HD double pm_epnp_rt(const PmEpnp& e, const double betas[4], double R[3][3], double t[3]) {
    double cc[4][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, pc[PM_N][3];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            for (int k = 0; k < 3; ++k) cc[j][k] += betas[i] * e.ut[i][3 * j + k];
    for (int i = 0; i < PM_N; ++i)
        for (int j = 0; j < 3; ++j)
            pc[i][j] = e.alpha[i][0] * cc[0][j] + e.alpha[i][1] * cc[1][j] + e.alpha[i][2] * cc[2][j] + e.alpha[i][3] * cc[3][j];
    if (pc[0][2] < 0.0)                                       // solve_for_sign
        for (int i = 0; i < PM_N; ++i)
            for (int j = 0; j < 3; ++j) pc[i][j] = -pc[i][j];
    double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
    for (int i = 0; i < PM_N; ++i)
        for (int j = 0; j < 3; ++j) { pc0[j] += pc[i][j]; pw0[j] += e.pw[i][j]; }
    for (int j = 0; j < 3; ++j) { pc0[j] /= PM_N; pw0[j] /= PM_N; }
    double abt[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = 0; i < PM_N; ++i)
        for (int j = 0; j < 3; ++j)
            for (int k = 0; k < 3; ++k) abt[j][k] += (pc[i][j] - pc0[j]) * (e.pw[i][k] - pw0[k]);
    if (!pm_procrustes(abt, R)) return INFINITY;
    for (int j = 0; j < 3; ++j) t[j] = pc0[j] - pm_dot3(R[j], pw0);
    double sum = 0.0;
    for (int i = 0; i < PM_N; ++i) {
        const double Xc = pm_dot3(R[0], e.pw[i]) + t[0], Yc = pm_dot3(R[1], e.pw[i]) + t[1], iz = 1.0 / (pm_dot3(R[2], e.pw[i]) + t[2]);
        const double du = e.us[i][0] - (e.uc + e.fu * Xc * iz), dv = e.us[i][1] - (e.vc + e.fv * Yc * iz);
        sum += sqrt(du * du + dv * dv);
    }
    const double err = sum / PM_N;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            if (!pm_finite(R[i][j])) return INFINITY;
    return pm_finite(err) && pm_finite(t[0]) && pm_finite(t[1]) && pm_finite(t[2]) ? err : INFINITY;
}

// epnp::gauss_newton: 5 steps on the 6 x 4 system of the four betas
PM_HD void pm_gauss_newton(const PmEpnp& e, double b[4]) {
    for (int it = 0; it < 5; ++it) {
        double A[6 * 4], r[6], x[4];
        for (int i = 0; i < 6; ++i) {
            const double* L = e.L[i];
            A[4 * i + 0] = 2 * L[0] * b[0] + L[1] * b[1] + L[3] * b[2] + L[6] * b[3];
            A[4 * i + 1] = L[1] * b[0] + 2 * L[2] * b[1] + L[4] * b[2] + L[7] * b[3];
            A[4 * i + 2] = L[3] * b[0] + L[4] * b[1] + 2 * L[5] * b[2] + L[8] * b[3];
            A[4 * i + 3] = L[6] * b[0] + L[7] * b[1] + L[8] * b[2] + 2 * L[9] * b[3];
            r[i] = e.rho[i] - (L[0] * b[0] * b[0] + L[1] * b[0] * b[1] + L[2] * b[1] * b[1] + L[3] * b[0] * b[2] + L[4] * b[1] * b[2] +
                               L[5] * b[2] * b[2] + L[6] * b[0] * b[3] + L[7] * b[1] * b[3] + L[8] * b[2] * b[3] + L[9] * b[3] * b[3]);
        }
        if (!pm_lsq6<4>(A, r, x)) return;
        for (int i = 0; i < 4; ++i) b[i] += x[i];
    }
}

// EPnP on PM_N correspondences: X world points, uv pixels, K = (fx, fy, cx, cy).  R row-major, t.  False: no pose.
PM_HD bool pm_epnp(const double X[PM_N][3], const double uv[PM_N][2], double fx, double fy, double cx, double cy, double Rout[9], double tout[3]) {
    PmEpnp e;
    e.fu = fx; e.fv = fy; e.uc = cx; e.vc = cy;
    for (int i = 0; i < PM_N; ++i) {
        for (int j = 0; j < 3; ++j) e.pw[i][j] = X[i][j];
        e.us[i][0] = uv[i][0]; e.us[i][1] = uv[i][1];
    }
    // 1. control points
    for (int j = 0; j < 3; ++j) {
        double s = 0.0;
        for (int i = 0; i < PM_N; ++i) s += e.pw[i][j];
        e.cw[0][j] = s / PM_N;
    }
    double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, E3[9];
    for (int i = 0; i < PM_N; ++i)
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) S[3 * a + b] += (e.pw[i][a] - e.cw[0][a]) * (e.pw[i][b] - e.cw[0][b]);
    pm_jacobi<3>(S, E3);
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2 - i; ++j)
            if (S[4 * o[j]] < S[4 * o[j + 1]]) { const int tmp = o[j]; o[j] = o[j + 1]; o[j + 1] = tmp; }
    const double l0 = S[4 * o[0]], l2 = S[4 * o[2]];
    // coincident, collinear or coplanar points: a control point collapses onto c0 and alpha is undefined
    if (!(l0 > 0.0) || !(l0 < 1e300) || !(l2 > 1e-12 * l0)) return false;
    double kk[3];
    for (int c = 0; c < 3; ++c) {
        kk[c] = sqrt(S[4 * o[c]] / PM_N);
        for (int j = 0; j < 3; ++j) e.cw[c + 1][j] = e.cw[0][j] + kk[c] * E3[3 * j + o[c]];
    }
    // 2. barycentric coordinates: the control frame is orthogonal, so CC^-1 (p - c0) = (e_c . (p - c0)) / k_c
    for (int i = 0; i < PM_N; ++i) {
        const double d[3] = {e.pw[i][0] - e.cw[0][0], e.pw[i][1] - e.cw[0][1], e.pw[i][2] - e.cw[0][2]};
        for (int c = 0; c < 3; ++c) e.alpha[i][c + 1] = (E3[o[c]] * d[0] + E3[3 + o[c]] * d[1] + E3[6 + o[c]] * d[2]) / kk[c];
        e.alpha[i][0] = 1.0 - e.alpha[i][1] - e.alpha[i][2] - e.alpha[i][3];
    }
    // 3. M^T M and its null space
    double MtM[144], V[144];
    for (int q = 0; q < 144; ++q) MtM[q] = 0.0;
    for (int i = 0; i < PM_N; ++i) {
        double m1[12], m2[12];
        for (int c = 0; c < 4; ++c) {
            const double a = e.alpha[i][c];
            m1[3 * c] = a * fx; m1[3 * c + 1] = 0.0; m1[3 * c + 2] = a * (cx - e.us[i][0]);
            m2[3 * c] = 0.0; m2[3 * c + 1] = a * fy; m2[3 * c + 2] = a * (cy - e.us[i][1]);
        }
        for (int a = 0; a < 12; ++a)
            for (int b = 0; b < 12; ++b) MtM[12 * a + b] += m1[a] * m1[b] + m2[a] * m2[b];
    }
    pm_jacobi<12>(MtM, V);
    int ord[12];
    for (int i = 0; i < 12; ++i) ord[i] = i;
    for (int i = 0; i < 4; ++i)                              // the 4 smallest eigenvalues, ascending
        for (int j = i + 1; j < 12; ++j)
            if (MtM[13 * ord[j]] < MtM[13 * ord[i]]) { const int tmp = ord[i]; ord[i] = ord[j]; ord[j] = tmp; }
    for (int i = 0; i < 4; ++i)
        for (int k = 0; k < 12; ++k) e.ut[i][k] = V[12 * k + ord[i]];
    // L (6 x 10) and rho: epnp::compute_L_6x10, compute_rho
    double dv[4][6][3];
    for (int i = 0; i < 4; ++i) {
        int a = 0, b = 1;
        for (int j = 0; j < 6; ++j) {
            for (int k = 0; k < 3; ++k) dv[i][j][k] = e.ut[i][3 * a + k] - e.ut[i][3 * b + k];
            if (++b > 3) { ++a; b = a + 1; }
        }
    }
    for (int i = 0; i < 6; ++i) {
        double* row = e.L[i];
        row[0] = pm_dot3(dv[0][i], dv[0][i]);
        row[1] = 2.0 * pm_dot3(dv[0][i], dv[1][i]);
        row[2] = pm_dot3(dv[1][i], dv[1][i]);
        row[3] = 2.0 * pm_dot3(dv[0][i], dv[2][i]);
        row[4] = 2.0 * pm_dot3(dv[1][i], dv[2][i]);
        row[5] = pm_dot3(dv[2][i], dv[2][i]);
        row[6] = 2.0 * pm_dot3(dv[0][i], dv[3][i]);
        row[7] = 2.0 * pm_dot3(dv[1][i], dv[3][i]);
        row[8] = 2.0 * pm_dot3(dv[2][i], dv[3][i]);
        row[9] = pm_dot3(dv[3][i], dv[3][i]);
    }
    {
        int j = 0;
        for (int a = 0; a < 4; ++a)
            for (int b = a + 1; b < 4; ++b, ++j) {
                const double d0 = e.cw[a][0] - e.cw[b][0], d1 = e.cw[a][1] - e.cw[b][1], d2 = e.cw[a][2] - e.cw[b][2];
                e.rho[j] = d0 * d0 + d1 * d1 + d2 * d2;
            }
    }
    // 4.-6. the three initialisations, Gauss-Newton, R and t; the lowest reprojection error wins (the first on a tie)
    double best = INFINITY;
    for (int N = 1; N <= 3; ++N) {
        double betas[4] = {0, 0, 0, 0}, A[6 * 5], x[5];
        bool ok;
        if (N == 1) {                                          // [B11 B12 B13 B14]
            for (int i = 0; i < 6; ++i) { A[4 * i] = e.L[i][0]; A[4 * i + 1] = e.L[i][1]; A[4 * i + 2] = e.L[i][3]; A[4 * i + 3] = e.L[i][6]; }
            ok = pm_lsq6<4>(A, e.rho, x);
            if (ok) {
                const double s = x[0] < 0 ? -1.0 : 1.0;
                betas[0] = sqrt(s * x[0]);
                betas[1] = s * x[1] / betas[0]; betas[2] = s * x[2] / betas[0]; betas[3] = s * x[3] / betas[0];
            }
        } else if (N == 2) {                                   // [B11 B12 B22]
            for (int i = 0; i < 6; ++i) { A[3 * i] = e.L[i][0]; A[3 * i + 1] = e.L[i][1]; A[3 * i + 2] = e.L[i][2]; }
            ok = pm_lsq6<3>(A, e.rho, x);
            if (ok) {
                if (x[0] < 0) { betas[0] = sqrt(-x[0]); betas[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0; }
                else { betas[0] = sqrt(x[0]); betas[1] = x[2] > 0 ? sqrt(x[2]) : 0.0; }
                if (x[1] < 0) betas[0] = -betas[0];
            }
        } else {                                               // [B11 B12 B22 B13 B23]
            for (int i = 0; i < 6; ++i)
                for (int c = 0; c < 5; ++c) A[5 * i + c] = e.L[i][c];
            ok = pm_lsq6<5>(A, e.rho, x);
            if (ok) {
                if (x[0] < 0) { betas[0] = sqrt(-x[0]); betas[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0; }
                else { betas[0] = sqrt(x[0]); betas[1] = x[2] > 0 ? sqrt(x[2]) : 0.0; }
                if (x[1] < 0) betas[0] = -betas[0];
                betas[2] = x[3] / betas[0];
            }
        }
        if (!ok || !pm_finite(betas[0]) || !pm_finite(betas[1]) || !pm_finite(betas[2]) || !pm_finite(betas[3])) continue;
        pm_gauss_newton(e, betas);
        double R[3][3], t[3];
        const double err = pm_epnp_rt(e, betas, R, t);
        if (err < best) {
            best = err;
            for (int i = 0; i < 3; ++i) { tout[i] = t[i]; for (int j = 0; j < 3; ++j) Rout[3 * i + j] = R[i][j]; }
        }
    }
    return best < INFINITY;
}

// Angle-axis of a rotation matrix (row-major) through its unit quaternion: accurate at every angle, including 0 and pi.
PM_HD void pm_rotmat_to_aa(const double* R, double* w) {
    const double tr = R[0] + R[4] + R[8];
    double q0, q1, q2, q3;                                     // w, x, y, z
    if (tr >= R[0] && tr >= R[4] && tr >= R[8]) {
        const double s = sqrt(1.0 + tr) * 2.0;
        q0 = 0.25 * s; q1 = (R[7] - R[5]) / s; q2 = (R[2] - R[6]) / s; q3 = (R[3] - R[1]) / s;
    } else if (R[0] >= R[4] && R[0] >= R[8]) {
        const double s = sqrt(1.0 + R[0] - R[4] - R[8]) * 2.0;
        q0 = (R[7] - R[5]) / s; q1 = 0.25 * s; q2 = (R[1] + R[3]) / s; q3 = (R[2] + R[6]) / s;
    } else if (R[4] >= R[8]) {
        const double s = sqrt(1.0 + R[4] - R[0] - R[8]) * 2.0;
        q0 = (R[2] - R[6]) / s; q1 = (R[1] + R[3]) / s; q2 = 0.25 * s; q3 = (R[5] + R[7]) / s;
    } else {
        const double s = sqrt(1.0 + R[8] - R[0] - R[4]) * 2.0;
        q0 = (R[3] - R[1]) / s; q1 = (R[2] + R[6]) / s; q2 = (R[5] + R[7]) / s; q3 = 0.25 * s;
    }
    const double sn = sqrt(q1 * q1 + q2 * q2 + q3 * q3);
    double k = 2.0;
    if (sn > 0.0) k = 2.0 * (q0 < 0.0 ? atan2(-sn, -q0) : atan2(sn, q0)) / sn;
    w[0] = k * q1; w[1] = k * q2; w[2] = k * q3;
}
