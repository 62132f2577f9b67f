// homography_math.cuh -- per-sample and per-pair arithmetic of the homography RANSAC (homography.cu), the algorithm of
// cv::findHomography(RANSAC) in OpenCV 4.x (calib3d fundam.cpp, ptsetreg.cpp, levmarq.cpp):
//   * cv::RNG, seeded with (uint64)-1 on every call, and getSubset: four indices drawn one after another, an index that
//     repeats an earlier one redrawn; the quad is rejected (and four new indices drawn) when the last point is collinear with
//     two earlier ones in either image, or when the four triples disagree in orientation between the images;
//   * the normalised 4-point / least-squares DLT of HomographyEstimatorCallback::runKernel: 9 x 9 L^T L, the eigenvector of
//     its smallest eigenvalue (cyclic Jacobi here), de-normalised and scaled to h22 = 1;
//   * the pieces of the Levenberg-Marquardt refinement (LMSolverImpl on h00..h21): residuals and Jacobian of one
//     correspondence, the 8 x 8 solves, the step-control rule.
// The decisions that must match OpenCV bit for bit (the random stream, the subset checks) are written without FMA
// contraction; the rest only has to agree to rounding.
// __host__ __device__, so tests compile the very same code with g++ and compare it with the numpy restatement and cv2.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define HM_HD __host__ __device__ __forceinline__
#else
#define HM_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define HM_MUL(a, b) __dmul_rn(a, b)
#define HM_ADD(a, b) __dadd_rn(a, b)
#define HM_SUB(a, b) __dsub_rn(a, b)
#else
#define HM_MUL(a, b) ((a) * (b))
#define HM_ADD(a, b) ((a) + (b))
#define HM_SUB(a, b) ((a) - (b))
#endif

constexpr int HM_SUBSET_ATTEMPTS = 10000;     // RANSACPointSetRegistrator::run -> getSubset(..., 10000)

// ---- cv::RNG -------------------------------------------------------------------------------------------------------------
HM_HD uint32_t hm_rng_next(uint64_t& s) {
    s = (uint64_t)(uint32_t)s * 4164903690ull + (s >> 32);
    return (uint32_t)s;
}
HM_HD int hm_rng_uniform(uint64_t& s, int n) { return (int)(hm_rng_next(s) % (uint32_t)n); }

// ---- subset checks (HomographyEstimatorCallback::checkSubset) -----------------------------------------------------------
// haveCollinearPoints for the last of four points; p = x0 y0 x1 y1 ...  The differences are float, as in OpenCV.
HM_HD bool hm_collinear4(const float* p) {
    for (int j = 0; j < 3; ++j) {
        const float fx1 = p[2 * j] - p[6], fy1 = p[2 * j + 1] - p[7];
        const double dx1 = fx1, dy1 = fy1;
        for (int k = 0; k < j; ++k) {
            const float fx2 = p[2 * k] - p[6], fy2 = p[2 * k + 1] - p[7];
            const double dx2 = fx2, dy2 = fy2;
            const double lhs = fabs(HM_SUB(HM_MUL(dx2, dy1), HM_MUL(dy2, dx1)));
            const double rhs = HM_MUL((double)FLT_EPSILON, HM_ADD(HM_ADD(HM_ADD(fabs(dx1), fabs(dy1)), fabs(dx2)), fabs(dy2)));
            if (lhs <= rhs) return true;
        }
    }
    return false;
}
// determinant of the rows (x, y, 1) of points t0, t1, t2 (cv::determinant of a Matx33d)
HM_HD double hm_det3(const float* p, int t0, int t1, int t2) {
    const double a00 = p[2 * t0], a01 = p[2 * t0 + 1], a10 = p[2 * t1], a11 = p[2 * t1 + 1], a20 = p[2 * t2], a21 = p[2 * t2 + 1];
    // a02 = a12 = a22 = 1
    const double m0 = HM_SUB(a11, a21), m1 = HM_SUB(a10, a20), m2 = HM_SUB(HM_MUL(a10, a21), HM_MUL(a20, a11));
    return HM_ADD(HM_SUB(HM_MUL(a00, m0), HM_MUL(a01, m1)), m2);
}
HM_HD bool hm_subset_ok(const float* s, const float* d) {
    if (hm_collinear4(s) || hm_collinear4(d)) return false;
    const int tt[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {1, 3, 0}};
    int negative = 0;
    for (int i = 0; i < 4; ++i)
        negative += HM_MUL(hm_det3(s, tt[i][0], tt[i][1], tt[i][2]), hm_det3(d, tt[i][0], tt[i][1], tt[i][2])) < 0.0 ? 1 : 0;
    return negative == 0 || negative == 4;
}

// getSubset: draws into idx[4] and returns true, or false after HM_SUBSET_ATTEMPTS rejected quads.  a, b = x y x y ...
HM_HD bool hm_draw_subset(uint64_t& s, int n, const float* a, const float* b, int idx[4]) {
    for (int attempt = 0; attempt < HM_SUBSET_ATTEMPTS; ++attempt) {
        float qa[8], qb[8];
        for (int i = 0; i < 4; ++i) {
            int v;
            for (;;) {
                v = hm_rng_uniform(s, n);
                bool dup = false;
                for (int k = 0; k < i; ++k) dup |= idx[k] == v;
                if (!dup) break;
            }
            idx[i] = v;
            qa[2 * i] = a[2 * v]; qa[2 * i + 1] = a[2 * v + 1];
            qb[2 * i] = b[2 * v]; qb[2 * i + 1] = b[2 * v + 1];
        }
        if (hm_subset_ok(qa, qb)) return true;
    }
    return false;
}

// ---- normalised DLT (HomographyEstimatorCallback::runKernel) ------------------------------------------------------------
// Normalisation of a correspondence set: centroids c and scales s = count / sum |p - c| per axis (M = source, m = destination).
struct HmNorm { double cMx, cMy, cmx, cmy, sMx, sMy, smx, smy; };

// from the sums of the coordinates and of the absolute deviations; false (no model) when a deviation sum is below DBL_EPSILON
HM_HD bool hm_norm_finish(int count, const double dev[4], HmNorm& nm) {
    if (fabs(dev[0]) < DBL_EPSILON || fabs(dev[1]) < DBL_EPSILON || fabs(dev[2]) < DBL_EPSILON || fabs(dev[3]) < DBL_EPSILON) return false;
    nm.sMx = count / dev[0]; nm.sMy = count / dev[1]; nm.smx = count / dev[2]; nm.smy = count / dev[3];
    return true;
}

// adds the two rows of one correspondence to the upper triangle of L^T L, packed row by row (45 entries)
HM_HD void hm_ltl_add(const HmNorm& nm, float Mx, float My, float mx, float my, double* L) {
    const double x = ((double)mx - nm.cmx) * nm.smx, y = ((double)my - nm.cmy) * nm.smy;
    const double X = ((double)Mx - nm.cMx) * nm.sMx, Y = ((double)My - nm.cMy) * nm.sMy;
    const double Lx[9] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y, -x};
    const double Ly[9] = {0, 0, 0, X, Y, 1, -y * X, -y * Y, -y};
    int o = 0;
    for (int j = 0; j < 9; ++j)
        for (int k = j; k < 9; ++k) L[o++] += Lx[j] * Lx[k] + Ly[j] * Ly[k];
}

// eigenvector v of the smallest eigenvalue of the symmetric 9 x 9 matrix A (row-major, destroyed): cyclic Jacobi
HM_HD void hm_jacobi_min9(double* A, double* v) {
    double V[81];
    for (int i = 0; i < 81; ++i) V[i] = (i % 10 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < 8; ++p)
            for (int q = p + 1; q < 9; ++q) {
                const double apq = A[9 * p + q];
                if (apq == 0.0) continue;
                const double app = A[9 * p + p], aqq = A[9 * q + q], g = 100.0 * fabs(apq);
                if (fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) { A[9 * p + q] = A[9 * q + p] = 0.0; continue; }
                rotated = true;
                const double theta = (aqq - app) / (2.0 * apq);
                const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 9; ++k) {          // columns: A G
                    const double akp = A[9 * k + p], akq = A[9 * k + q];
                    A[9 * k + p] = c * akp - s * akq; A[9 * k + q] = s * akp + c * akq;
                }
                for (int k = 0; k < 9; ++k) {          // rows: G^T (A G)
                    const double apk = A[9 * p + k], aqk = A[9 * q + k];
                    A[9 * p + k] = c * apk - s * aqk; A[9 * q + k] = s * apk + c * aqk;
                }
                A[9 * p + q] = A[9 * q + p] = 0.0;
                for (int k = 0; k < 9; ++k) {
                    const double vkp = V[9 * k + p], vkq = V[9 * k + q];
                    V[9 * k + p] = c * vkp - s * vkq; V[9 * k + q] = s * vkp + c * vkq;
                }
            }
        if (!rotated) break;
    }
    int m = 0;
    for (int i = 1; i < 9; ++i)
        if (A[10 * i] < A[10 * m]) m = i;
    for (int k = 0; k < 9; ++k) v[k] = V[9 * k + m];
}

// H = invHnorm * h * Hnorm2 / (.)_22 from the packed upper triangle of L^T L (destroyed into a full matrix on the way)
HM_HD void hm_solve_ltl(const double* Lpacked, const HmNorm& nm, double* H) {
    double A[81], h[9];
    int o = 0;
    for (int j = 0; j < 9; ++j)
        for (int k = j; k < 9; ++k) { A[9 * j + k] = A[9 * k + j] = Lpacked[o++]; }
    hm_jacobi_min9(A, h);
    const double iN[9] = {1.0 / nm.smx, 0, nm.cmx, 0, 1.0 / nm.smy, nm.cmy, 0, 0, 1};
    const double N2[9] = {nm.sMx, 0, -nm.cMx * nm.sMx, 0, nm.sMy, -nm.cMy * nm.sMy, 0, 0, 1};
    double T[9], H0[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) T[3 * r + c] = iN[3 * r] * h[c] + iN[3 * r + 1] * h[3 + c] + iN[3 * r + 2] * h[6 + c];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) H0[3 * r + c] = T[3 * r] * N2[c] + T[3 * r + 1] * N2[3 + c] + T[3 * r + 2] * N2[6 + c];
    const double s = 1.0 / H0[8];
    for (int k = 0; k < 9; ++k) H[k] = H0[k] * s;
    H[8] = 1.0;
}

// the whole kernel on count correspondences held in registers / local memory (the 4-point minimal case); false = no model
HM_HD bool hm_kernel(const float* M, const float* m, int count, double* H) {
    HmNorm nm;
    double sum[4] = {0, 0, 0, 0}, dev[4] = {0, 0, 0, 0};
    for (int i = 0; i < count; ++i) { sum[0] += M[2 * i]; sum[1] += M[2 * i + 1]; sum[2] += m[2 * i]; sum[3] += m[2 * i + 1]; }
    nm.cMx = sum[0] / count; nm.cMy = sum[1] / count; nm.cmx = sum[2] / count; nm.cmy = sum[3] / count;
    for (int i = 0; i < count; ++i) {
        dev[0] += fabs(M[2 * i] - nm.cMx); dev[1] += fabs(M[2 * i + 1] - nm.cMy);
        dev[2] += fabs(m[2 * i] - nm.cmx); dev[3] += fabs(m[2 * i + 1] - nm.cmy);
    }
    if (!hm_norm_finish(count, dev, nm)) return false;
    double L[45];
    for (int k = 0; k < 45; ++k) L[k] = 0.0;
    for (int i = 0; i < count; ++i) hm_ltl_add(nm, M[2 * i], M[2 * i + 1], m[2 * i], m[2 * i + 1], L);
    hm_solve_ltl(L, nm, H);
    return true;
}

// ---- Levenberg-Marquardt refinement (LMSolverImpl, HomographyRefineCallback) --------------------------------------------
// residuals r = (H X) / w - x of one correspondence and, when J != nullptr, their 2 x 8 Jacobian
HM_HD void hm_residual(const double* h, float fMx, float fMy, float fmx, float fmy, double r[2], double* J) {
    const double Mx = fMx, My = fMy;
    double ww = h[6] * Mx + h[7] * My + 1.0;
    ww = fabs(ww) > DBL_EPSILON ? 1.0 / ww : 0.0;
    const double xi = (h[0] * Mx + h[1] * My + h[2]) * ww, yi = (h[3] * Mx + h[4] * My + h[5]) * ww;
    r[0] = xi - (double)fmx; r[1] = yi - (double)fmy;
    if (!J) return;
    J[0] = Mx * ww; J[1] = My * ww; J[2] = ww; J[3] = J[4] = J[5] = 0.0; J[6] = -Mx * ww * xi; J[7] = -My * ww * xi;
    J[8] = J[9] = J[10] = 0.0; J[11] = Mx * ww; J[12] = My * ww; J[13] = ww; J[14] = -Mx * ww * yi; J[15] = -My * ww * yi;
}

// normal-equation terms of one correspondence added to acc: A = J^T J upper triangle (36, packed), v = J^T r (8), S = r.r
constexpr int HM_LM_TERMS = 36 + 8 + 1;
HM_HD void hm_lm_add(const double* h, float Mx, float My, float mx, float my, double* acc, double& rinf) {
    double r[2], J[16];
    hm_residual(h, Mx, My, mx, my, r, J);
    int o = 0;
    for (int j = 0; j < 8; ++j)
        for (int k = j; k < 8; ++k) acc[o++] += J[j] * J[k] + J[8 + j] * J[8 + k];
    for (int j = 0; j < 8; ++j) acc[36 + j] += J[j] * r[0] + J[8 + j] * r[1];
    acc[44] += r[0] * r[0] + r[1] * r[1];
    rinf = fmax(rinf, fmax(fabs(r[0]), fabs(r[1])));
}

// x = A^-1 b for a symmetric 8 x 8 A (row-major); Gaussian elimination with partial pivoting; a zero pivot leaves x_k = 0
HM_HD void hm_solve8(const double* A0, const double* b0, double* x) {
    double A[64], b[8];
    for (int k = 0; k < 64; ++k) A[k] = A0[k];
    for (int k = 0; k < 8; ++k) b[k] = b0[k];
    for (int c = 0; c < 8; ++c) {
        int p = c;
        for (int r = c + 1; r < 8; ++r)
            if (fabs(A[8 * r + c]) > fabs(A[8 * p + c])) p = r;
        if (p != c) {
            for (int k = 0; k < 8; ++k) { const double t = A[8 * c + k]; A[8 * c + k] = A[8 * p + k]; A[8 * p + k] = t; }
            const double t = b[c]; b[c] = b[p]; b[p] = t;
        }
        if (A[8 * c + c] == 0.0) continue;
        for (int r = c + 1; r < 8; ++r) {
            const double f = A[8 * r + c] / A[8 * c + c];
            for (int k = c; k < 8; ++k) A[8 * r + k] -= f * A[8 * c + k];
            b[r] -= f * b[c];
        }
    }
    for (int c = 7; c >= 0; --c) {
        double s = b[c];
        for (int k = c + 1; k < 8; ++k) s -= A[8 * c + k] * x[k];
        x[c] = A[8 * c + c] != 0.0 ? s / A[8 * c + c] : 0.0;
    }
}

// LMSolverImpl's state between block reductions.  A, v, S, rinf are at x; D = diag(A) at the start.
struct HmLm {
    double x[8], xd[8], d[8], A[64], v[8], D[8];
    double S, rinf, lambda, lc;
    int iter;
};

HM_HD void hm_lm_load(HmLm& st, const double* acc, double rinf) {
    int o = 0;
    for (int j = 0; j < 8; ++j)
        for (int k = j; k < 8; ++k) { st.A[8 * j + k] = st.A[8 * k + j] = acc[o++]; }
    for (int j = 0; j < 8; ++j) st.v[j] = acc[36 + j];
    st.S = acc[44]; st.rinf = rinf;
}
HM_HD void hm_lm_init(HmLm& st, const double* H, const double* acc, double rinf) {
    for (int k = 0; k < 8; ++k) st.x[k] = H[k];
    hm_lm_load(st, acc, rinf);
    for (int k = 0; k < 8; ++k) st.D[k] = st.A[9 * k];
    st.lambda = 1.0; st.lc = 0.75; st.iter = 0;
}
// the trial step: d = (A + lambda D)^-1 v, xd = x - d
HM_HD void hm_lm_propose(HmLm& st) {
    double Ap[64];
    for (int k = 0; k < 64; ++k) Ap[k] = st.A[k];
    for (int k = 0; k < 8; ++k) Ap[9 * k] += st.lambda * st.D[k];
    hm_solve8(Ap, st.v, st.d);
    for (int k = 0; k < 8; ++k) st.xd[k] = st.x[k] - st.d[k];
}
// the step control given the cost Sd at xd; returns true when the step is accepted (the caller then re-evaluates A, v, S, rinf
// at the new x with hm_lm_load)
HM_HD bool hm_lm_update(HmLm& st, double Sd) {
    double dS = 0.0, t = 0.0;
    for (int i = 0; i < 8; ++i) {
        double Ad = 0.0;
        for (int k = 0; k < 8; ++k) Ad += st.A[8 * i + k] * st.d[k];
        dS += st.d[i] * (2.0 * st.v[i] - Ad);
        t += st.d[i] * st.v[i];
    }
    const double R = (st.S - Sd) / (fabs(dS) > DBL_EPSILON ? dS : 1.0);
    if (R > 0.75) {
        st.lambda *= 0.5;
        if (st.lambda < st.lc) st.lambda = 0.0;
    } else if (R < 0.25) {
        double nu = (Sd - st.S) / (fabs(t) > DBL_EPSILON ? t : 1.0) + 2.0;
        nu = fmin(fmax(nu, 2.0), 10.0);
        if (st.lambda == 0.0) {
            double maxval = DBL_EPSILON;
            for (int k = 0; k < 8; ++k) {
                double e[8], col[8];
                for (int q = 0; q < 8; ++q) e[q] = q == k ? 1.0 : 0.0;
                hm_solve8(st.A, e, col);
                maxval = fmax(maxval, fabs(col[k]));
            }
            st.lambda = st.lc = 1.0 / maxval;
            nu *= 0.5;
        }
        st.lambda *= nu;
    }
    if (!(Sd < st.S)) return false;
    for (int k = 0; k < 8; ++k) st.x[k] = st.xd[k];
    return true;
}
// after the (possibly re-evaluated) state of this iteration: continue?
HM_HD bool hm_lm_proceed(HmLm& st, int max_iters) {
    ++st.iter;
    double dinf = 0.0;
    for (int k = 0; k < 8; ++k) dinf = fmax(dinf, fabs(st.d[k]));
    return st.iter < max_iters && dinf >= FLT_EPSILON && st.rinf >= FLT_EPSILON;
}
