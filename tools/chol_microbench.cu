// tools/chol_microbench.cu -- K4 in isolation: the streaming dataflow Cholesky kernel on an SPD matrix of the
// reduced-camera-system size, checked against a host factorisation, with the critical-path timeline from its %globaltimer
// trace; then the cluster and the single-CTA back-solves on its factor, checked against a host solve.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -o tools/_build/chol_microbench tools/chol_microbench.cu
// Usage: chol_microbench [cams=100] [reps=20]
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../sfm-toy-library_b200/csrc/chol.cuh"

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

// task t of chol_stream_kernel -> tile (i, c); merged tasks also factor (i, i)
static void decode(int t, int nbk, int& i, int& c, bool& merged) {
    merged = false;
    if (t == 0) { i = c = 0; return; }
    int rem = t - 1, cnt = nbk - 1; c = 0;
    while (rem >= cnt) { rem -= cnt; ++c; cnt = nbk - 1 - c; }
    i = c + 1 + rem; merged = rem == 0;
}

int main(int argc, char** argv) {
    const int nc = argc > 1 ? atoi(argv[1]) : 100, reps = argc > 2 ? atoi(argv[2]) : 20;
    const int n = 6 * nc + 1, npad = ((n + 1) + NB - 1) / NB * NB, nbk = npad / NB;
    std::vector<double> A((size_t)npad * npad, 0.0), L;
    srand(7);
    for (int r = 0; r < n; ++r) for (int c = 0; c <= r; ++c) A[(size_t)r * npad + c] = (r == c) ? n + 1.0 : (rand() / (double)RAND_MAX * 2 - 1);
    for (int c = 0; c < n; ++c) A[(size_t)n * npad + c] = rand() / (double)RAND_MAX * 2 - 1;
    for (int r = n + 1; r < npad; ++r) A[(size_t)r * npad + r] = 1.0;
    // host reference (same conventions: pivots >= n are 1 with a zero column)
    L = A;
    for (int j = 0; j < npad; ++j) {
        if (j >= n) { L[(size_t)j * npad + j] = 1.0; for (int r = j + 1; r < npad; ++r) L[(size_t)r * npad + j] = 0.0; continue; }
        double d = L[(size_t)j * npad + j];
        for (int k = 0; k < j; ++k) d -= L[(size_t)j * npad + k] * L[(size_t)j * npad + k];
        const double ljj = std::sqrt(d); L[(size_t)j * npad + j] = ljj;
        for (int r = j + 1; r < npad; ++r) {
            double v = L[(size_t)r * npad + j];
            for (int k = 0; k < j; ++k) v -= L[(size_t)r * npad + k] * L[(size_t)j * npad + k];
            L[(size_t)r * npad + j] = v / ljj;
        }
    }
    double *dA0, *dA, *ddinv, *dLinv, *dx; int* dfail; unsigned* dready; uint4* dprogress; unsigned long long* dtrace;
    const size_t bytes = sizeof(double) * npad * npad;
    CK(cudaMalloc(&dA0, bytes)); CK(cudaMalloc(&dA, bytes)); CK(cudaMalloc(&ddinv, 8 * npad)); CK(cudaMalloc(&dfail, 16));
    CK(cudaMalloc(&dready, 4 * nbk * nbk)); CK(cudaMalloc(&dLinv, 8 * (size_t)npad * NB)); CK(cudaMalloc(&dx, 8 * npad)); CK(cudaMalloc(&dtrace, 64 * (size_t)nbk * nbk));
    CK(cudaMemcpy(dA0, A.data(), bytes, cudaMemcpyHostToDevice)); CK(cudaMemset(dfail, 0, 16)); CK(cudaMemset(dready, 0, 4 * nbk * nbk)); CK(cudaMalloc(&dprogress, chol_ll_bytes(nbk))); CK(cudaMemset(dprogress, 0, chol_ll_bytes(nbk)));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    unsigned epoch = 0;
    std::vector<double> out((size_t)npad * npad);
    std::vector<unsigned long long> tr((size_t)8 * nbk * nbk);
    {
        int per_sm = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chol_stream_kernel, CS_THREADS, 0));
        const int ntasks = chol_stream_tasks(nbk), grid = std::min(ntasks, per_sm * prop.multiProcessorCount);
        float total = 0, best = 1e30f;
        for (int rep = 0; rep < reps + 2; ++rep) {
            const bool traced = rep == reps + 1;
            CK(cudaMemcpy(dA, dA0, bytes, cudaMemcpyDeviceToDevice));
            if (traced) CK(cudaMemset(dtrace, 0, 64 * (size_t)nbk * nbk));
            CK(cudaDeviceSynchronize());
            CK(cudaEventRecord(e0));
            chol_stream_kernel<<<grid, CS_THREADS>>>(dA, npad, n, nbk, ntasks, ddinv, dfail, dready, dprogress, ++epoch, dLinv, traced ? dtrace : nullptr);
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep >= 1 && !traced) { total += ms; best = std::min(best, ms); }
        }
        CK(cudaMemcpy(out.data(), dA, bytes, cudaMemcpyDeviceToHost));
        int fail[4]; CK(cudaMemcpy(fail, dfail, 16, cudaMemcpyDeviceToHost));
        double err = 0, ref = 0;
        for (int r = 0; r <= n; ++r) for (int c = 0; c <= std::min(r, n - 1); ++c) {
            err = std::max(err, std::fabs(out[(size_t)r * npad + c] - L[(size_t)r * npad + c])); ref = std::max(ref, std::fabs(L[(size_t)r * npad + c]));
        }
        printf("{\"variant\": \"%s\", \"cams\": %d, \"n\": %d, \"tile_rows\": %d, \"grid\": %d, \"tasks\": %d, \"avg_us\": %.1f, \"best_us\": %.1f, \"max_abs_err\": %.3e, \"max_abs_L\": %.3e, \"fail\": %d}\n",
               "streaming dataflow (DMMA updates)", nc, n, nbk, grid, ntasks, total / reps * 1e3, best * 1e3, err, ref, fail[0]);
        CK(cudaMemcpy(tr.data(), dtrace, 64 * (size_t)ntasks, cudaMemcpyDeviceToHost));
        // critical path: per diagonal tile j, the stamps of the task that factors it
        unsigned long long t_start = ~0ull;
        for (int t = 0; t < ntasks; ++t) t_start = std::min(t_start, tr[(size_t)t * 8]);
        std::vector<double> pub(nbk, 0), seen(nbk, 0), solved(nbk, 0), pubx(nbk, 0), fact(nbk, 0), upd(nbk, 0), fstart(nbk, 0);
        for (int t = 0; t < ntasks; ++t) {
            int i, c; bool merged;
            decode(t, nbk, i, c, merged);
            const unsigned long long* e = &tr[(size_t)t * 8];
            auto us = [&](int slot) { return e[slot] ? (e[slot] - t_start) * 1e-3 : 0.0; };
            if (i == c || merged) { pub[i] = us(6); fact[i] = us(5); upd[i] = us(1); fstart[i] = us(7); }
            if (merged) { seen[i] = us(2); solved[i] = us(3); pubx[i] = us(4); }
        }
#ifdef CHOL_FINE_TRACE
        {
            unsigned long long f[64]; CK(cudaMemcpyFromSymbol(f, g_chol_fine, sizeof f));
            printf("  fine trace of the factorisation of tile 10 (cycles since entry): entry 0");
            for (int k = 1; k < 36; ++k) if (f[k]) printf("%s %lld", (k % 4) == 1 ? "\n    round owner_in/owner_out/after_barrier/[after_update]:" : "", (long long)(f[k] - f[0]));
            printf("\n");
            unsigned long long g[64]; CK(cudaMemcpyFromSymbol(g, g_chol_fine2, sizeof g));
            for (int r = 0; r < 8; ++r) printf("    round %d owner section, cycles: shuffles->pivots %lld, column vectors %lld, stores %lld\n", r,
                                               (long long)(g[r * 8 + 1] - g[r * 8]), (long long)(g[r * 8 + 2] - g[r * 8 + 1]), (long long)(g[r * 8 + 3] - g[r * 8 + 2]));
        }
#endif
        printf("  j  published(j,j) us   step   | updates_done  diag_seen  solved  x_published  factor_start  factored\n");
        for (int j = 0; j < nbk; ++j) {
            printf("  %2d %10.2f %10.2f | %8.2f %8.2f %8.2f %8.2f %8.2f %8.2f\n", j, pub[j], j ? pub[j] - pub[j - 1] : pub[j], upd[j], seen[j], solved[j], pubx[j], fstart[j], fact[j]);
        }
    }
    // ---- both back substitutions on the factor left by the last run (Linv from the dataflow kernel)
    {
        std::vector<double> xr(n, 0.0), xg(n);
        for (int r = n - 1; r >= 0; --r) {
            double v = L[(size_t)n * npad + r];
            for (int k = r + 1; k < n; ++k) v -= L[(size_t)k * npad + r] * xr[k];
            xr[r] = v / L[(size_t)r * npad + r];
        }
        {   // cluster variant (BS_CLUSTER CTAs)
            const size_t cs = chol_backsolve_cluster_smem(n); const int cthreads = chol_backsolve_cluster_threads(n);
            CK(cudaFuncSetAttribute(chol_backsolve_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs));
            float total = 0;
            for (int rep = 0; rep < reps + 1; ++rep) {
                CK(cudaMemset(dx, 0, 8 * npad)); CK(cudaDeviceSynchronize());
                CK(cudaEventRecord(e0));
                chol_backsolve_cluster_kernel<<<BS_CLUSTER, cthreads, cs>>>(dA, dLinv, npad, n, dx, dfail);
                CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
                float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (rep) total += ms;
            }
            CK(cudaMemcpy(xg.data(), dx, 8 * n, cudaMemcpyDeviceToHost));
            double err = 0, ref = 0;
            for (int r = 0; r < n; ++r) { err = std::max(err, std::fabs(xg[r] - xr[r])); ref = std::max(ref, std::fabs(xr[r])); }
            int fl[4]; CK(cudaMemcpy(fl, dfail, 16, cudaMemcpyDeviceToHost));
            printf("{\"variant\": \"backsolve cluster of %d CTAs x %d threads, %zu B smem\", \"avg_us\": %.1f, \"max_abs_err\": %.3e, \"max_abs_x\": %.3e, \"fail\": %d}\n", BS_CLUSTER, cthreads, cs, total / reps * 1e3, err, ref, fl[0]);
        }
        {   // single CTA
            const size_t sm = chol_backsolve_smem(npad);
            float total = 0;
            for (int rep = 0; rep < reps + 1; ++rep) {
                CK(cudaMemset(dx, 0, 8 * npad)); CK(cudaDeviceSynchronize());
                CK(cudaEventRecord(e0));
                chol_backsolve_kernel<<<1, 640, sm>>>(dA, dLinv, npad, n, dx);
                CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
                float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (rep) total += ms;
            }
            CK(cudaMemcpy(xg.data(), dx, 8 * n, cudaMemcpyDeviceToHost));
            double err = 0, ref = 0;
            for (int r = 0; r < n; ++r) { err = std::max(err, std::fabs(xg[r] - xr[r])); ref = std::max(ref, std::fabs(xr[r])); }
            printf("{\"variant\": \"backsolve single CTA x 640 threads, %zu B smem\", \"avg_us\": %.1f, \"max_abs_err\": %.3e, \"max_abs_x\": %.3e}\n", sm, total / reps * 1e3, err, ref);
        }
    }
    return 0;
}
