// tools/fp64_peak.cu -- measured fp64 issue peaks of the device: DFMA (CUDA cores) and DMMA m8n8k4 (mma.sync f64).
// These are the denominators for the "fp64" side of the BA roofline (MEASURED_PEAKS.json only carries HBM and bf16).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/_build/fp64_peak tools/fp64_peak.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void __launch_bounds__(256) dfma_kernel(double* out, int iters, double a, double b) {
    double x[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = threadIdx.x * 1e-3 + i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = fma(x[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += x[i];
    if (s == 12345.678) out[0] = s;
}

__global__ void __launch_bounds__(256) dmma_kernel(double* out, int iters, double a, double b) {
    double c[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) { c[i][0] = threadIdx.x; c[i][1] = i; }
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) s += c[i][0] + c[i][1];
    if (s == 12345.678) out[0] = s;
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    double* d; cudaMalloc(&d, 8);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20000, blocks = p.multiProcessorCount * 8;
    for (int which = 0; which < 2; ++which) {
        float best = 1e30f;
        for (int rep = 0; rep < 5; ++rep) {
            cudaEventRecord(e0);
            if (which == 0) dfma_kernel<<<blocks, 256>>>(d, iters, 0.999999, 1e-9); else dmma_kernel<<<blocks, 256>>>(d, iters, 0.5, 0.25);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
        }
        const double fl = which == 0 ? 2.0 * 8 * iters * 256.0 * blocks : 2.0 * 256 * 4 * iters * 8.0 * blocks;   // dmma: 8*8*4 FMA per warp instr
        printf("{\"kernel\": \"%s\", \"ms\": %.3f, \"tflops\": %.2f, \"sms\": %d}\n", which == 0 ? "dfma" : "dmma_m8n8k4", best, fl / best * 1e-9, p.multiProcessorCount);
    }
    printf("cuda error: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
