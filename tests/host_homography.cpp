// tests/host_homography.cpp -- TEST HARNESS: runs the __host__ __device__ arithmetic of csrc/homography_math.cuh (cv::RNG,
// getSubset, the normalised DLT, the Levenberg-Marquardt step control) on the CPU, in the order homography.cu runs it.
// Not part of the product library.
#include "../sfm-toy-library_b200/csrc/homography_math.cuh"
extern "C" {
// `count` consecutive subsets of one RANSAC run from the seeded generator -> idx [count][4]; returns how many were found before
// getSubset gave up (count when it never did)
int host_draw_subsets(const float* a, const float* b, int n, int count, int* idx) {
    uint64_t s = ~0ull;
    for (int k = 0; k < count; ++k)
        if (!hm_draw_subset(s, n, a, b, idx + 4 * k)) return k;
    return count;
}
// the DLT on `count` correspondences -> H [9]; 0 = no model
int host_kernel(const float* M, const float* m, int count, double* H) { return hm_kernel(M, m, count, H) ? 1 : 0; }
// Levenberg-Marquardt from H on `count` correspondences -> Hout [9]; returns the iterations run
int host_refine(const float* M, const float* m, int count, const double* H, int max_iters, double* Hout) {
    double acc[HM_LM_TERMS], rinf = 0.0;
    auto eval = [&](const double* h) {
        for (int k = 0; k < HM_LM_TERMS; ++k) acc[k] = 0.0;
        rinf = 0.0;
        for (int i = 0; i < count; ++i) hm_lm_add(h, M[2 * i], M[2 * i + 1], m[2 * i], m[2 * i + 1], acc, rinf);
    };
    HmLm st;
    eval(H);
    hm_lm_init(st, H, acc, rinf);
    for (;;) {
        hm_lm_propose(st);
        double Sd = 0.0;
        for (int i = 0; i < count; ++i) {
            double r[2];
            hm_residual(st.xd, M[2 * i], M[2 * i + 1], m[2 * i], m[2 * i + 1], r, nullptr);
            Sd += r[0] * r[0] + r[1] * r[1];
        }
        if (hm_lm_update(st, Sd)) { eval(st.x); hm_lm_load(st, acc, rinf); }
        if (!hm_lm_proceed(st, max_iters)) break;
    }
    for (int k = 0; k < 8; ++k) Hout[k] = st.x[k];
    Hout[8] = 1.0;
    return st.iter;
}
}
