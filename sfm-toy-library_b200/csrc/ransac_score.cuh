// ransac_score.cuh -- the RANSAC error formulas, inlier rule and scoring / best / mask kernels of ransac.cu, shared with the
// essential-matrix and homography RANSACs (essential.cu, homography.cu), which score their device-made hypotheses with the very
// same arithmetic, together with the sample budget of OpenCV's sequential loop.
// See ransac.cu for which OpenCV computeError callback each formula mirrors.
#pragma once
#include <cfloat>
#include <cmath>
#include "common.cuh"

namespace {

constexpr int RS_THREADS = 256;

struct Model { double m[12]; };      // 3x3 (homography / essential) or 3x4 pose, row-major

__device__ __forceinline__ float err_homography(const double* H, float x, float y, float X, float Y) {
    // no FMA contraction: the CPU code is plain float mul/add in this order
    const float h0 = (float)H[0], h1 = (float)H[1], h2 = (float)H[2], h3 = (float)H[3], h4 = (float)H[4], h5 = (float)H[5], h6 = (float)H[6], h7 = (float)H[7];
    const float ww = __fdiv_rn(1.f, __fadd_rn(__fadd_rn(__fmul_rn(h6, x), __fmul_rn(h7, y)), 1.f));
    const float dx = __fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(h0, x), __fmul_rn(h1, y)), h2), ww), X);
    const float dy = __fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(h3, x), __fmul_rn(h4, y)), h5), ww), Y);
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}
__device__ __forceinline__ float err_essential(const double* E, double x1, double y1, double x2, double y2) {
    // Ex1 = E * (x1, y1, 1), Etx2 = E^T * (x2, y2, 1)
    const double e0 = __dadd_rn(__dadd_rn(__dmul_rn(E[0], x1), __dmul_rn(E[1], y1)), E[2]);
    const double e1 = __dadd_rn(__dadd_rn(__dmul_rn(E[3], x1), __dmul_rn(E[4], y1)), E[5]);
    const double e2 = __dadd_rn(__dadd_rn(__dmul_rn(E[6], x1), __dmul_rn(E[7], y1)), E[8]);
    const double t0 = __dadd_rn(__dadd_rn(__dmul_rn(E[0], x2), __dmul_rn(E[3], y2)), E[6]);
    const double t1 = __dadd_rn(__dadd_rn(__dmul_rn(E[1], x2), __dmul_rn(E[4], y2)), E[7]);
    const double x2tEx1 = __dadd_rn(__dadd_rn(__dmul_rn(x2, e0), __dmul_rn(y2, e1)), e2);
    const double den = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e0, e0), __dmul_rn(e1, e1)), __dmul_rn(t0, t0)), __dmul_rn(t1, t1));
    return (float)(__dmul_rn(x2tEx1, x2tEx1) / den);
}
__device__ __forceinline__ float err_pose(const double* P, const double* K, float X, float Y, float Z, float u, float v) {
    const double x = P[0] * X + P[1] * Y + P[2] * Z + P[3], y = P[4] * X + P[5] * Y + P[6] * Z + P[7], z = P[8] * X + P[9] * Y + P[10] * Z + P[11];
    const double iz = z != 0.0 ? 1.0 / z : 1.0;          // cv::projectPoints: z = z ? 1./z : 1
    const float pu = (float)(K[0] * (x * iz) + K[2]), pv = (float)(K[4] * (y * iz) + K[5]);
    const float dx = __fsub_rn(u, pu), dy = __fsub_rn(v, pv);
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

// model: 0 homography, 1 essential (a, b already normalised doubles? no: float pixels, normalised here with f, cx, cy in aux), 2 pose
template <int MODEL>
__device__ __forceinline__ bool is_inlier(const double* M, const double* aux, const float* __restrict__ a, const float* __restrict__ b, int i, float t2) {
    if (MODEL == 0) return err_homography(M, a[2 * i], a[2 * i + 1], b[2 * i], b[2 * i + 1]) <= t2;
    if (MODEL == 1) {
        // cv::findEssentialMat(points, focal, pp): points converted to double and normalised (x - cx) / f before the estimator
        const double f = aux[0], cx = aux[1], cy = aux[2];
        return err_essential(M, ((double)a[2 * i] - cx) / f, ((double)a[2 * i + 1] - cy) / f, ((double)b[2 * i] - cx) / f, ((double)b[2 * i + 1] - cy) / f) <= t2;
    }
    return err_pose(M, aux, a[3 * i], a[3 * i + 1], a[3 * i + 2], b[2 * i], b[2 * i + 1]) <= t2;
}

template <int MODEL>
__global__ void __launch_bounds__(RS_THREADS) ransac_score_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, const Model* __restrict__ hyp,
                                                                  const double* __restrict__ aux, float t2, int per_block, int32_t* __restrict__ counts) {
    __shared__ double M[12], A[9];
    __shared__ int wsum[RS_THREADS / 32];
    if (threadIdx.x < 12) M[threadIdx.x] = hyp[blockIdx.y].m[threadIdx.x];
    if (threadIdx.x < 9) A[threadIdx.x] = aux[threadIdx.x];
    __syncthreads();
    const int begin = blockIdx.x * per_block, end = min(n, begin + per_block);
    int c = 0;
    for (int i = begin + threadIdx.x; i < end; i += RS_THREADS) c += is_inlier<MODEL>(M, A, a, b, i, t2) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < RS_THREADS / 32; ++w) s += wsum[w];
        if (s) atomicAdd(counts + blockIdx.y, s);
    }
}

// best hypothesis = most inliers, ties -> lowest index; single CTA
__global__ void __launch_bounds__(1024) ransac_best_kernel(const int32_t* __restrict__ counts, int nh, int32_t* __restrict__ best) {
    __shared__ long long red[32];
    long long key = -1;                                   // (count << 32) | (0x7fffffff - index): max = most inliers, lowest index
    for (int h = threadIdx.x; h < nh; h += 1024) { const long long k = ((long long)counts[h] << 32) | (long long)(0x7fffffff - h); key = k > key ? k : key; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const long long other = __shfl_xor_sync(0xffffffffu, key, o); key = other > key ? other : key; }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = key;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 32; ++w) key = red[w] > key ? red[w] : key;
        best[0] = nh > 0 ? 0x7fffffff - (int)(key & 0xffffffffLL) : -1;
        best[1] = nh > 0 ? (int)(key >> 32) : 0;
    }
}
template <int MODEL>
__global__ void __launch_bounds__(RS_THREADS) ransac_mask_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, const Model* __restrict__ hyp,
                                                                 const double* __restrict__ aux, float t2, const int32_t* __restrict__ best, uint8_t* __restrict__ mask) {
    const int h = best[0];
    const int i = blockIdx.x * RS_THREADS + threadIdx.x;
    if (i >= n) return;
    if (h < 0) { mask[i] = 0; return; }
    double M[12], A[9];
#pragma unroll
    for (int k = 0; k < 12; ++k) M[k] = hyp[h].m[k];
#pragma unroll
    for (int k = 0; k < 9; ++k) A[k] = aux[k];
    mask[i] = is_inlier<MODEL>(M, A, a, b, i, t2) ? 1 : 0;
}

// RANSACUpdateNumIters (OpenCV calib3d ptsetreg.cpp), cvRound = round half to even
__device__ int ransac_update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = fmin(fmax(p, 0.0), 1.0);
    ep = fmin(fmax(ep, 0.0), 1.0);
    double num = fmax(1.0 - p, DBL_MIN);
    double denom = 1.0 - pow(1.0 - ep, (double)model_points);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : __double2int_rn(num / denom);
}

}  // namespace
