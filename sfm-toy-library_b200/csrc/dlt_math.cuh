// dlt_math.cuh -- smallest right singular vector of the 4 x 4 two-view DLT matrix (cv::triangulatePoints), shared by the
// triangulation stage (triangulate.cu) and the cheirality test of the pose recovery (essential.cu).
// __host__ __device__, so that tests/ can run the very same code on the CPU against an exact reference.
#pragma once
#include <cfloat>
#include <cmath>

#if defined(__CUDACC__)
#define DLT_HD __host__ __device__ __forceinline__
#else
#define DLT_HD inline
using std::isfinite;   // <cmath> declares the others in the global namespace too
#endif

namespace {

// One Hestenes rotation between columns I and J of A (4 rows), accumulating V.
#define SFM_JROT(I, J)                                                                                            \
    {                                                                                                             \
        const double p0 = A[0][I] * A[0][J] + A[1][I] * A[1][J] + A[2][I] * A[2][J] + A[3][I] * A[3][J];          \
        const double a = nrm[I], b = nrm[J];                                                                      \
        if (fabs(p0) > eps * sqrt(a * b)) {                                                                       \
            const double p = 2.0 * p0, beta = a - b, gamma = hypot(p, beta);                                      \
            double c, s;                                                                                          \
            if (beta < 0) { const double delta = (gamma - beta) * 0.5; s = sqrt(delta / gamma); c = p / (gamma * s * 2.0); } \
            else { c = sqrt((gamma + beta) / (gamma * 2.0)); s = p / (gamma * c * 2.0); }                         \
            double na = 0, nb = 0;                                                                                \
            _Pragma("unroll") for (int k = 0; k < 4; ++k) {                                                      \
                const double t0 = c * A[k][I] + s * A[k][J], t1 = -s * A[k][I] + c * A[k][J];                     \
                A[k][I] = t0; A[k][J] = t1; na = fma(t0, t0, na); nb = fma(t1, t1, nb);                           \
                const double v0 = c * V[k][I] + s * V[k][J], v1 = -s * V[k][I] + c * V[k][J];                     \
                V[k][I] = v0; V[k][J] = v1;                                                                       \
            }                                                                                                     \
            nrm[I] = na; nrm[J] = nb; rotated = true;                                                             \
        }                                                                                                         \
    }

DLT_HD void null_vector_4x4(double A[4][4], double X[4]) {
    double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    double nrm[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) nrm[j] = A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j] + A[3][j] * A[3][j];
    const double eps = DBL_EPSILON * 10;
    for (int sweep = 0; sweep < 30; ++sweep) {
        bool rotated = false;
        SFM_JROT(0, 1) SFM_JROT(0, 2) SFM_JROT(0, 3) SFM_JROT(1, 2) SFM_JROT(1, 3) SFM_JROT(2, 3)
        if (!rotated) break;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) nrm[j] = A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j] + A[3][j] * A[3][j];
    // smallest singular value; among equal norms the last column (cv::SVD sorts descending, takes the last row of Vt)
    double best = nrm[0];
#pragma unroll
    for (int k = 0; k < 4; ++k) X[k] = V[k][0];
#pragma unroll
    for (int j = 1; j < 4; ++j) {
        if (nrm[j] <= best) {
            best = nrm[j];
#pragma unroll
            for (int k = 0; k < 4; ++k) X[k] = V[k][j];
        }
    }
}

// ---- fast path for the smallest right singular vector --------------------------------------------------------------
// For a well-conditioned two-view DLT the 4x4 matrix B = A^T A has one eigenvalue far below the other three.  Its
// characteristic polynomial p(x) = x^4 - c3 x^3 + c2 x^2 - c1 x + c0 has only real roots, so Newton's iteration started
// at 0 climbs monotonically to the smallest one; the eigenvector is then a column of adj(B - x I) (rank-3 matrix: every
// column of the adjugate is a multiple of the null vector; the column with the largest diagonal cofactor is used).
// ~600 flops instead of ~5000 for the Jacobi SVD.  The result is verified (residual of the eigen-equation); anything
// suspicious falls back to the Jacobi routine above, which is the reference-faithful algorithm.
DLT_HD double det3(double a, double b, double c, double d, double e, double f, double g, double h, double i) {
    return a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
}
struct Sym4 { double c00, c01, c02, c03, c11, c12, c13, c22, c23, c33; };
struct Adj4 { double k00, k01, k02, k03, k11, k12, k13, k22, k23, k33; };
DLT_HD void adjugate_sym4(const Sym4& m, Adj4& k) {
    k.k00 = det3(m.c11, m.c12, m.c13, m.c12, m.c22, m.c23, m.c13, m.c23, m.c33);
    k.k01 = -det3(m.c01, m.c12, m.c13, m.c02, m.c22, m.c23, m.c03, m.c23, m.c33);
    k.k02 = det3(m.c01, m.c11, m.c13, m.c02, m.c12, m.c23, m.c03, m.c13, m.c33);
    k.k03 = -det3(m.c01, m.c11, m.c12, m.c02, m.c12, m.c22, m.c03, m.c13, m.c23);
    k.k11 = det3(m.c00, m.c02, m.c03, m.c02, m.c22, m.c23, m.c03, m.c23, m.c33);
    k.k12 = -det3(m.c00, m.c01, m.c03, m.c02, m.c12, m.c23, m.c03, m.c13, m.c33);
    k.k13 = det3(m.c00, m.c01, m.c02, m.c02, m.c12, m.c22, m.c03, m.c13, m.c23);
    k.k22 = det3(m.c00, m.c01, m.c03, m.c01, m.c11, m.c13, m.c03, m.c13, m.c33);
    k.k23 = -det3(m.c00, m.c01, m.c02, m.c01, m.c11, m.c12, m.c03, m.c13, m.c23);
    k.k33 = det3(m.c00, m.c01, m.c02, m.c01, m.c11, m.c12, m.c02, m.c12, m.c22);
}
DLT_HD bool null_vector_fast(const double A[4][4], double X[4]) {
    Sym4 B;
    B.c00 = A[0][0] * A[0][0] + A[1][0] * A[1][0] + A[2][0] * A[2][0] + A[3][0] * A[3][0];
    B.c01 = A[0][0] * A[0][1] + A[1][0] * A[1][1] + A[2][0] * A[2][1] + A[3][0] * A[3][1];
    B.c02 = A[0][0] * A[0][2] + A[1][0] * A[1][2] + A[2][0] * A[2][2] + A[3][0] * A[3][2];
    B.c03 = A[0][0] * A[0][3] + A[1][0] * A[1][3] + A[2][0] * A[2][3] + A[3][0] * A[3][3];
    B.c11 = A[0][1] * A[0][1] + A[1][1] * A[1][1] + A[2][1] * A[2][1] + A[3][1] * A[3][1];
    B.c12 = A[0][1] * A[0][2] + A[1][1] * A[1][2] + A[2][1] * A[2][2] + A[3][1] * A[3][2];
    B.c13 = A[0][1] * A[0][3] + A[1][1] * A[1][3] + A[2][1] * A[2][3] + A[3][1] * A[3][3];
    B.c22 = A[0][2] * A[0][2] + A[1][2] * A[1][2] + A[2][2] * A[2][2] + A[3][2] * A[3][2];
    B.c23 = A[0][2] * A[0][3] + A[1][2] * A[1][3] + A[2][2] * A[2][3] + A[3][2] * A[3][3];
    B.c33 = A[0][3] * A[0][3] + A[1][3] * A[1][3] + A[2][3] * A[2][3] + A[3][3] * A[3][3];
    const double c3 = B.c00 + B.c11 + B.c22 + B.c33;
    if (!(c3 > 0.0) || !isfinite(c3)) return false;
    Adj4 K;
    adjugate_sym4(B, K);
    const double c1 = K.k00 + K.k11 + K.k22 + K.k33;
    const double c0 = B.c00 * K.k00 + B.c01 * K.k01 + B.c02 * K.k02 + B.c03 * K.k03;
    const double c2 = (B.c00 * B.c11 - B.c01 * B.c01) + (B.c00 * B.c22 - B.c02 * B.c02) + (B.c00 * B.c33 - B.c03 * B.c03) +
                      (B.c11 * B.c22 - B.c12 * B.c12) + (B.c11 * B.c33 - B.c13 * B.c13) + (B.c22 * B.c33 - B.c23 * B.c23);
    if (!(c1 > 0.0)) return false;
    double x = 0.0;
    bool conv = false;
#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        const double p = (((x - c3) * x + c2) * x - c1) * x + c0;
        const double dp = ((4.0 * x - 3.0 * c3) * x + 2.0 * c2) * x - c1;
        if (!(dp < 0.0)) return false;
        const double step = p / dp;                   // <= 0 while below the root
        x -= step;
        if (fabs(step) <= 1e-15 * c3) { conv = true; break; }
    }
    if (!conv || !(x >= -1e-12 * c3)) return false;
    Sym4 C = B;
    C.c00 -= x; C.c11 -= x; C.c22 -= x; C.c33 -= x;
    adjugate_sym4(C, K);
    const double a0 = fabs(K.k00), a1 = fabs(K.k11), a2 = fabs(K.k22), a3 = fabs(K.k33);
    double v0, v1, v2, v3;
    if (a0 >= a1 && a0 >= a2 && a0 >= a3) { v0 = K.k00; v1 = K.k01; v2 = K.k02; v3 = K.k03; }
    else if (a1 >= a2 && a1 >= a3) { v0 = K.k01; v1 = K.k11; v2 = K.k12; v3 = K.k13; }
    else if (a2 >= a3) { v0 = K.k02; v1 = K.k12; v2 = K.k22; v3 = K.k23; }
    else { v0 = K.k03; v1 = K.k13; v2 = K.k23; v3 = K.k33; }
    const double vn = fmax(fmax(fabs(v0), fabs(v1)), fmax(fabs(v2), fabs(v3)));
    if (!(vn > 0.0) || !isfinite(vn)) return false;
    // verify (B - x I) v = 0 and that x is well separated from the next eigenvalue: p'(x) = -prod_{i<4}(lambda_i - x)
    const double r0 = C.c00 * v0 + C.c01 * v1 + C.c02 * v2 + C.c03 * v3, r1 = C.c01 * v0 + C.c11 * v1 + C.c12 * v2 + C.c13 * v3;
    const double r2 = C.c02 * v0 + C.c12 * v1 + C.c22 * v2 + C.c23 * v3, r3 = C.c03 * v0 + C.c13 * v1 + C.c23 * v2 + C.c33 * v3;
    const double rn = fmax(fmax(fabs(r0), fabs(r1)), fmax(fabs(r2), fabs(r3)));
    const double dpx = ((4.0 * x - 3.0 * c3) * x + 2.0 * c2) * x - c1;
    // gap estimate: |p'(x)| >= (lambda_3 - x) * (c3/4)^2-ish; demand lambda_3 - x >= 1e-7 * c3 (conservative), residual tiny
    if (!(-dpx >= 1e-7 * c3 * c3 * c3 * (1.0 / 64.0)) || !(rn <= 1e-11 * c3 * vn)) return false;
    X[0] = v0; X[1] = v1; X[2] = v2; X[3] = v3;
    return true;
}

}  // namespace
