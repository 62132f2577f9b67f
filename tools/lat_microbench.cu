// tools/lat_microbench.cu -- dependent-issue latencies (cycles) of what the tile factorisation's pivot chain is made of:
// DFMA, DMUL, the refined reciprocal square root, a shuffle, a shared-memory round trip, a 128-thread named barrier.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/_build/lat_microbench tools/lat_microbench.cu
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ double rsqrt_fast(double d) {
    double y; asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    const double t = y * y, e = fma(-d, t, 1.0), p2 = fma(e, 0.375, 0.5), q = y * e;
    return fma(p2, q, y);
}

constexpr int N = 256;
__global__ void lat_kernel(double* out, long long* cyc, double seed) {
    __shared__ double sm[128];
    const int lane = threadIdx.x & 31;
    double x = seed + lane * 1e-9, acc = 0;
    long long t0, t1;
    // 0: DFMA
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = fma(x, 1.0000001, 1e-9);
    t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0; acc += x;
    // 1: DMUL
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = x * 1.0000001;
    t1 = clock64(); if (threadIdx.x == 0) cyc[1] = t1 - t0; acc += x;
    // 2: refined rsqrt
    x = 2.0 + lane;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = rsqrt_fast(x) + 1.5;
    t1 = clock64(); if (threadIdx.x == 0) cyc[2] = t1 - t0; acc += x;
    // 3: MUFU seed alone (+ the add that closes the chain)
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) { double y; asm volatile("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x)); x = y + 1.5; }
    t1 = clock64(); if (threadIdx.x == 0) cyc[3] = t1 - t0; acc += x;
    // 4: shuffle of a double
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = __shfl_sync(0xffffffffu, x, (lane + 1) & 31);
    t1 = clock64(); if (threadIdx.x == 0) cyc[4] = t1 - t0; acc += x;
    // 5: shared-memory round trip (STS + LDS of another lane's slot, one warp)
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) { sm[threadIdx.x] = x; __syncwarp(); x = sm[threadIdx.x ^ 1]; __syncwarp(); }
    t1 = clock64(); if (threadIdx.x == 0) cyc[5] = t1 - t0; acc += x;
    // 6: named barrier over the 128 threads
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("bar.sync 1, 128;" ::: "memory");
    t1 = clock64(); if (threadIdx.x == 0) cyc[6] = t1 - t0;
    // 7: STS + barrier + LDS (the publish step of the factorisation)
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) { sm[threadIdx.x] = x; asm volatile("bar.sync 1, 128;" ::: "memory"); x = sm[(threadIdx.x + 32) & 127]; }
    t1 = clock64(); if (threadIdx.x == 0) cyc[7] = t1 - t0; acc += x;
    // 8: DSETP + select closing a chain
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = (x > 0.5 && x < 1e300) ? x * 1.0000001 : 1.0;
    t1 = clock64(); if (threadIdx.x == 0) cyc[8] = t1 - t0; acc += x;
    out[threadIdx.x] = acc;
}

int main() {
    double* out; long long* cyc;
    cudaMalloc(&out, 128 * 8); cudaMalloc(&cyc, 16 * 8); cudaMemset(cyc, 0, 128);
    for (int r = 0; r < 3; ++r) lat_kernel<<<1, 128>>>(out, cyc, 1.0);
    long long h[16];
    if (cudaMemcpy(h, cyc, 128, cudaMemcpyDeviceToHost) != cudaSuccess) { printf("failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
    const char* names[] = {"DFMA", "DMUL", "rsqrt refined (+DADD)", "MUFU.RSQ64H seed (+DADD)", "SHFL f64", "STS+LDS (warp)", "bar.sync 1,128",
                           "STS + bar + LDS", "DSETP x2 + select + DMUL"};
    for (int i = 0; i < 9; ++i) printf("%-28s %7.1f cycles\n", names[i], (double)h[i] / N);
    return 0;
}
