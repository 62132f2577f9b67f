// tools/red_microbench.cu -- measures the fp64 global-reduction (red.global.add.f64) throughput of the Schur
// accumulation pattern of ba_point_kernel on the target GPU, to size the design (DESIGN.md, "K3a accumulation").
// 200k points x 8 cameras (random, ascending) out of 100 -> 28 pair blocks x 36 doubles per point into a 1.45 MB S.
//   mode 0: coalesced, one entry per lane (32 consecutive doubles per RED instruction)         <- what K3a does
//   mode 1: one 6x6 block per lane (28 lanes busy, 36 RED instructions, each touching 28 different blocks)
//   mode 2: as mode 0 with plain stores instead of RED (upper bound of the store path)
//   mode 3: as mode 0 but every warp hits the SAME block (same-address contention)
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/_build/red_microbench tools/red_microbench.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <cuda_runtime.h>

__device__ __forceinline__ void red_add(double* p, double v) { asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ size_t blk_index(int i, int j, int nb) { return (size_t)i * nb - (size_t)i * (i - 1) / 2 + (j - i); }

template <int MODE>
__global__ void kern(const int* __restrict__ cams /*[np*8]*/, int np, int nb, double* __restrict__ S) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int p = warp; p < np; p += nwarps) {
        const int* c = cams + 8 * p;
        if (MODE == 1) {
            if (lane < 28) {
                int i = 0, rem = lane; while (rem >= 7 - i) { rem -= 7 - i; ++i; } const int j = i + 1 + rem;
                double* b = S + blk_index(c[i], c[j], nb) * 36;
#pragma unroll
                for (int e = 0; e < 36; ++e) red_add(b + e, 1e-9 * (e + lane));
            }
        } else {
            for (int e = lane; e < 28 * 36; e += 32) {
                const int pr = e / 36, ab = e - pr * 36;
                int i = 0, rem = pr; while (rem >= 7 - i) { rem -= 7 - i; ++i; } const int j = i + 1 + rem;
                double* dst = S + (MODE == 3 ? 0 : blk_index(c[i], c[j], nb) * 36) + ab;
                if (MODE == 2) *dst = 1e-9 * e; else red_add(dst, 1e-9 * e);
            }
        }
    }
}

int main() {
    const int np = 200000, nb = 100;
    std::vector<int> h(np * 8);
    srand(1);
    for (int p = 0; p < np; ++p) {
        int sel[8], n = 0;
        while (n < 8) { int c = rand() % nb; bool dup = false; for (int q = 0; q < n; ++q) dup |= sel[q] == c; if (!dup) sel[n++] = c; }
        std::sort(sel, sel + 8);
        for (int q = 0; q < 8; ++q) h[8 * p + q] = sel[q];
    }
    int* d_c; double* d_S; const size_t sn = (size_t)nb * (nb + 1) / 2 * 36;
    cudaMalloc(&d_c, sizeof(int) * h.size()); cudaMalloc(&d_S, sizeof(double) * sn);
    cudaMemcpy(d_c, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice); cudaMemset(d_S, 0, sizeof(double) * sn);
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const double entries = (double)np * 28 * 36;
    for (int mode = 0; mode < 4; ++mode) {
        for (int bps : {4, 8, 16}) {
            const int blocks = prop.multiProcessorCount * bps;
            float best = 1e9f;
            for (int rep = 0; rep < 5; ++rep) {
                cudaEventRecord(e0);
                if (mode == 0) kern<0><<<blocks, 128>>>(d_c, np, nb, d_S);
                else if (mode == 1) kern<1><<<blocks, 128>>>(d_c, np, nb, d_S);
                else if (mode == 2) kern<2><<<blocks, 128>>>(d_c, np, nb, d_S);
                else kern<3><<<blocks, 128>>>(d_c, np, nb, d_S);
                cudaEventRecord(e1); cudaEventSynchronize(e1);
                float ms; cudaEventElapsedTime(&ms, e0, e1); if (rep > 0 && ms < best) best = ms;
            }
            printf("mode %d blocks/SM %2d : %8.1f us  %.2f G entries/s  %.1f GB/s of 8-byte updates  (err %s)\n", mode, bps, best * 1e3,
                   entries / best * 1e-6, entries * 8 / best * 1e-6, cudaGetErrorString(cudaGetLastError()));
        }
    }
    return 0;
}
