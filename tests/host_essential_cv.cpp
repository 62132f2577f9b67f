// tests/host_essential_cv.cpp -- TEST HARNESS: runs the __host__ __device__ OpenCV sampler of csrc/essential_math.cuh
// (em_cv_samples over cv_rng.cuh) and the five-point solver on the CPU.  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/essential_math.cuh"
extern "C" {
// the first S samples for m correspondences -> out [S][5]
void host_cv_samples(int m, int S, int* out) { em_cv_samples(m, S, out); }
// the raw stream: `count` draws of rng.uniform(0, n) from cv::RNG((uint64)-1)
void host_cv_uniform(int n, int count, int* out) {
    uint64_t s = CV_RNG_SEED;
    for (int i = 0; i < count; ++i) out[i] = cv_rng_uniform(s, n);
}
// x1, x2 [ns][5][2] normalised coordinates -> E [ns][10][9], nsol [ns]
void host_five_point(const double* x1, const double* x2, int ns, double* E, int* nsol) {
    for (int s = 0; s < ns; ++s)
        nsol[s] = five_point_solve((const double(*)[2])(x1 + 10 * s), (const double(*)[2])(x2 + 10 * s), (double(*)[9])(E + 90 * s));
}
}
