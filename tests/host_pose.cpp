// tests/host_pose.cpp -- TEST HARNESS: runs the __host__ __device__ EPnP solver and rotation conversion of csrc/pose_math.cuh and the
// sequential RANSAC selection of csrc/ransac_select.cuh on the CPU.  Not part of the product library.
#include <cstdint>
#include "../sfm-toy-library_b200/csrc/pose_math.cuh"
#include "../sfm-toy-library_b200/csrc/ransac_select.cuh"
extern "C" {
// X [ns][5][3], uv [ns][5][2], K = (fx, fy, cx, cy) -> Rt [ns][12] row-major [R|t], ok [ns]
void host_epnp(const double* X, const double* uv, const double* K, int ns, double* Rt, int* ok) {
    for (int s = 0; s < ns; ++s) {
        double R[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, t[3] = {0, 0, 0};
        ok[s] = pm_epnp((const double(*)[3])(X + 15 * s), (const double(*)[2])(uv + 10 * s), K[0], K[1], K[2], K[3], R, t) ? 1 : 0;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) Rt[12 * s + 4 * r + c] = R[3 * r + c];
            Rt[12 * s + 4 * r + 3] = t[r];
        }
    }
}
void host_rotmat_to_aa(const double* R, double* w) { pm_rotmat_to_aa(R, w); }
// the device's loop: samples staged 32 at a time; nsol [S], counts [S * slots] -> out = (best slot, best count, samples visited)
void host_select(const int32_t* nsol, const int32_t* counts, int S, int slots, int n, int max_iters, double confidence, int model_points, int* out) {
    SeqSelect st;
    seq_select_begin(st, max_iters);
    for (int base = 0; base < S && st.iter < st.niters; base += 32) {
        const int k = S - base < 32 ? S - base : 32;
        seq_select_chunk(st, nsol + base, counts + (size_t)slots * base, slots, k, n, confidence, model_points, 0);
    }
    out[0] = st.best; out[1] = st.max_good; out[2] = st.iter;
}
int host_update_num_iters(double p, double ep, int model_points, int max_iters) { return ransac_update_num_iters(p, ep, model_points, max_iters); }
}
