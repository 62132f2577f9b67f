// tests/host_essential.cpp -- TEST HARNESS: runs the __host__ __device__ five-point solver, the sample drawing and the
// essential-matrix decomposition of csrc/essential_math.cuh on the CPU.  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/essential_math.cuh"
extern "C" {
// x1, x2 [ns][5][2] normalised coordinates -> E [ns][10][9], nsol [ns]
void host_five_point(const double* x1, const double* x2, int ns, double* E, int* nsol) {
    for (int s = 0; s < ns; ++s)
        nsol[s] = five_point_solve((const double(*)[2])(x1 + 10 * s), (const double(*)[2])(x2 + 10 * s), (double(*)[9])(E + 90 * s));
}
void host_sample(unsigned long long seed, int s, int n, int* idx) { em_sample(seed, (uint32_t)s, n, idx); }
int host_decompose(const double* E, double* R1, double* R2, double* t) { return em_decompose_essential(E, R1, R2, t) ? 1 : 0; }
int host_real_roots10(const double* p, double* roots) { return em_real_roots10(p, roots); }
}
