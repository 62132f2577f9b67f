// cv_rng.cuh -- OpenCV's random stream as RANSACPointSetRegistrator::run (calib3d ptsetreg.cpp, OpenCV 4.x) consumes it: a
// cv::RNG seeded with (uint64)-1 on every call, multiply-with-carry with the coefficient 4164903690, each draw the low 32 bits,
// rng.uniform(0, n) = draw % n; getSubset draws the indices of a sample one after another and redraws an index that repeats an
// earlier one of the same sample.  Integer arithmetic only, so host and device give the same bits.  Used by the homography RANSAC
// (homography_math.cuh, whose getSubset adds its own subset checks) and the essential-matrix RANSAC (essential.cu).
// __host__ __device__, so tests compile the very same code with g++.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define CV_RNG_HD __host__ __device__ __forceinline__
#else
#define CV_RNG_HD inline
#endif

constexpr uint64_t CV_RNG_SEED = ~0ull;      // cv::RNG rng((uint64)-1)

CV_RNG_HD uint32_t cv_rng_next(uint64_t& s) {
    s = (uint64_t)(uint32_t)s * 4164903690ull + (s >> 32);
    return (uint32_t)s;
}
CV_RNG_HD int cv_rng_uniform(uint64_t& s, int n) { return (int)(cv_rng_next(s) % (uint32_t)n); }

// K distinct indices in [0, n) into idx, in draw order; n >= K
template <int K>
CV_RNG_HD void cv_rng_distinct(uint64_t& s, int n, int idx[K]) {
    for (int i = 0; i < K; ++i) {
        int v;
        for (;;) {
            v = cv_rng_uniform(s, n);
            bool dup = false;
            for (int k = 0; k < i; ++k) dup |= idx[k] == v;
            if (!dup) break;
        }
        idx[i] = v;
    }
}
