// ransac_select.cuh -- the selection half of OpenCV's RANSAC (RANSACPointSetRegistrator::run and RANSACUpdateNumIters, OpenCV
// calib3d ptsetreg.cpp) over inlier counts already scored in sample order.  Shared by the essential-matrix RANSAC (up to 10
// solutions per sample) and the PnP RANSAC (one solution per sample); __host__ __device__, so tests compile the very same loop
// with g++ and compare it with their restatement of OpenCV's.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define RS_HD __host__ __device__ __forceinline__
#else
#define RS_HD inline
#endif

namespace {

// RANSACUpdateNumIters (OpenCV calib3d ptsetreg.cpp), cvRound = round half to even
RS_HD int ransac_update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = fmin(fmax(p, 0.0), 1.0);
    ep = fmin(fmax(ep, 0.0), 1.0);
    double num = fmax(1.0 - p, DBL_MIN);
    double denom = 1.0 - pow(1.0 - ep, (double)model_points);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
#if defined(__CUDA_ARCH__)
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : __double2int_rn(num / denom);
#else
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)nearbyint(num / denom);
#endif
}

// State of the sequential loop: sample budget, best solution (slot index, -1 = none), its count, samples visited.
struct SeqSelect {
    int niters, best, max_good, iter;
};

RS_HD void seq_select_begin(SeqSelect& st, int max_iters) {
    st.niters = max_iters > 1 ? max_iters : 1; st.best = -1; st.max_good = 0; st.iter = 0;
}

// The loop over the next k samples (st.iter, st.iter + 1, ...) of a set of n correspondences: sample j has nsol[j] solutions
// whose counts are counts[slots * j + q].  A solution replaces the best one only if its count exceeds max(best count,
// model_points - 1); every improvement recomputes the budget with RANSACUpdateNumIters(confidence, outlier ratio, model_points,
// budget); the loop stops at the budget, and a sample it enters is visited whole.  The best is recorded as slot
// slot_base + slots * (sample) + q.
RS_HD void seq_select_chunk(SeqSelect& st, const int32_t* nsol, const int32_t* counts, int slots, int k, int n, double confidence,
                            int model_points, int slot_base) {
    for (int j = 0; j < k && st.iter < st.niters; ++j, ++st.iter)
        for (int q = 0; q < nsol[j]; ++q) {
            const int g = counts[slots * j + q];
            if (g > (st.max_good > model_points - 1 ? st.max_good : model_points - 1)) {
                st.best = slot_base + slots * st.iter + q; st.max_good = g;
                st.niters = ransac_update_num_iters(confidence, (double)(n - g) / n, model_points, st.niters);
            }
        }
}

}  // namespace
