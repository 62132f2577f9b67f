// tests/host_dlt.cpp -- TEST HARNESS: runs the __host__ __device__ null-vector code of csrc/dlt_math.cuh on the CPU, both of its
// paths on every matrix.  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/dlt_math.cuh"
extern "C" {
// A [n][4][4] -> the closed form's vector vf [n][4] (zeros where it declines) and its decision ok [n]; the Jacobi vector vj [n][4]
void host_null_vectors(const double* A, int n, double* vf, int* ok, double* vj) {
    for (int i = 0; i < n; ++i) {
        double a[4][4], b[4][4], x[4] = {0, 0, 0, 0};
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) a[r][c] = b[r][c] = A[16 * i + 4 * r + c];
        ok[i] = null_vector_fast(a, x) ? 1 : 0;
        for (int k = 0; k < 4; ++k) vf[4 * i + k] = ok[i] ? x[k] : 0.0;
        null_vector_4x4(b, vj + 4 * i);
    }
}
}
