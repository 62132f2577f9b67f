// common.cuh -- context, error plumbing and device scratch shared by every stage of libsfmb200.so.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <string>
#include <vector>
#include <mutex>
#include <array>
#include <utility>

#include "../../include/sfmb200.h"
#include "host_pool.h"

// One growable device buffer + one pinned host buffer per purpose, reused across calls (cudaMalloc/cudaFree are
// milliseconds; the reference calls each stage many times per runSfM()).
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct PinBuf {
    void* p = nullptr; size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// bump allocator over a DevBuf: carve() after a single reserve()
struct Carver {
    char* base; size_t off = 0;
    explicit Carver(void* b) : base((char*)b) {}
    template <typename T> T* take(size_t n) {
        off = (off + 255) & ~size_t(255);
        T* r = (T*)(base + off); off += n * sizeof(T); return r;
    }
    static size_t pad(size_t bytes) { return (bytes + 255) & ~size_t(255); }
};

struct CommState;   // comm.cu

// Device / pinned workspace of one bundle-adjustment problem, kept by the context between problems: adjustBundle is called
// once per added view (SfM.cpp:350, :529) and the one-shot sfmb200_ba_solve would otherwise pay cudaMalloc / cudaFree /
// cudaMallocHost of several hundred MB on every call.  One problem at a time borrows it; further live problems allocate.
struct BAWorkspace {
    DevBuf mem, gmem, xbuf;
    PinBuf hpin;
    bool in_use = false;
    void release() { mem.release(); gmem.release(); xbuf.release(); hpin.release(); }
};

// Descriptor images kept resident between per-call matchFeatures invocations (match.cu): one arena of packed rows, one of
// expanded tensor-core operand blocks, bump-allocated, flushed whole when full.
struct MatchCacheEntry { const void* host; int rows; int desc_bytes; uint64_t hash; int row0; int blk0; };
struct MatchCache {
    DevBuf desc, exp;
    int width = 0;                       // padded descriptor width (bytes) of the rows in the arena
    int64_t rows_cap = 0, rows_used = 0;
    int blk_cap = 0, blk_used = 0;
    std::vector<MatchCacheEntry> entries;
    int64_t hits = 0, misses = 0;
    void release() { desc.release(); exp.release(); entries.clear(); rows_cap = rows_used = 0; blk_cap = blk_used = 0; }
};

// Device buffers of the last ORB extraction (orb.cu), kept for sfmb200_orb_download_level (stage-by-stage parity tests).
struct OrbLast { uint8_t *pyr = nullptr, *blur = nullptr, *score = nullptr; int slab = 0, nimg = 0, w = 0, h = 0, nfeatures = 0; };

// Device memory of one descriptor set (match.cu), kept by the context between sets: SfM::createFeatureMatchMatrix builds one set per run and
// a benchmark one per repetition -- cudaMalloc / cudaFree (a device-wide synchronisation each) cost more than matching 21 image pairs.
// One set at a time borrows it; further live sets allocate their own memory.
struct DescWorkspace {
    DevBuf desc, exp, norms;
    bool in_use = false;
    void release() { desc.release(); exp.release(); norms.release(); }
};

struct sfmb200_ctx {
    int device = 0;
    int sm_count = 0;
    int l2_bytes = 0;           // L2 cache size (sizes the L2-resident working sets of the bundle adjustment)
    cudaStream_t stream = nullptr;
    std::string err;
    int64_t launches = 0;
    std::mutex mu;              // matchFeatures is called from several host threads in the reference (SfM.cpp:173-211)
    DevBuf scratch;             // per-call device scratch (kernel workspace)
    DevBuf scratch2;            // per-call device scratch (stage outputs)
    PinBuf pinned;              // per-call pinned staging (results read-back)
    BAWorkspace ba_ws;          // cached bundle-adjustment workspace
    MatchCache mcache;          // descriptor images resident between per-call matchFeatures invocations
    DescWorkspace ds_ws;        // cached device memory of a descriptor set
    DevBuf orb_dev, orb_lists;  // ORB extraction: pyramids / score maps / candidates of a batch of images; key point lists
    PinBuf orb_pin_img, orb_pin_a, orb_pin_b, orb_pin_c;   // ORB extraction: pinned image staging / staging of the three host round trips
    double orb_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};            // host wall-clock of the phases of the last extraction (sfmb200_orb_last_timings)
    HostPool* pool = nullptr;   // host threads for the work that stays on the CPU (created on first use)
    OrbLast orb_last;
    cudaStream_t orb_stream = nullptr;            // the Gaussian blur of the pyramid runs beside the detection chain
    cudaStream_t orb_up = nullptr;                // image uploads run beside the detection of the images that have already landed
    std::vector<cudaEvent_t> orb_img_ev;          // "image s of the batch is on the device"
    cudaEvent_t orb_ev[2] = {nullptr, nullptr};   // pyramid ready / blur done
    bool tc_attr_set = false;   // cudaFuncSetAttribute(knn2_hamming_tc_kernel, max dynamic smem) done for THIS device
    // peer exchange buffers opened with cudaIpcOpenMemHandle, kept open across problems (the exchange buffer is part of the cached
    // BA workspace, so the one-shot solve sees the same handles on every call): handle bytes -> mapped base
    std::vector<std::pair<std::array<uint8_t, 64>, void*>> ipc_cache;
    CommState* comm = nullptr;
    int rank = 0, nranks = 1;
    DevBuf ess_trace;           // samples / solution counts / inlier counts of the last essential-matrix RANSAC (essential.cu)
    int ess_trace_samples = 0;
    DevBuf hg_trace;            // visited samples / counts of the last homography RANSAC with record_trace (homography.cu)
    int hg_trace_pairs = 0, hg_trace_stride = 0;
    std::vector<int32_t> hg_trace_visited;
    DevBuf jpeg_dev;                    // JPEG decoding (jpeg.cu): tables, entropy data, coefficients, planes, images of the last batch
    PinBuf jpeg_pin_up, jpeg_pin_down;  // its one upload and its one download
    int64_t jpeg_stats[7] = {0, 0, 0, 0, 0, 0, 0};   // sfmb200_jpeg_last_stats of the last batch
    DevBuf rz_dev;                      // image downscale (resize.cu): descriptors, taps, source and resized images of the last batch
    PinBuf rz_pin_up, rz_pin_down;      // its one upload and its one download
};

int sfmb200_fail(sfmb200_ctx* ctx, int code, const char* fmt, ...);

#define SFM_CUDA(ctx, call)                                                                              \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess)                                                                           \
            return sfmb200_fail((ctx), e_ == cudaErrorMemoryAllocation ? SFMB200_ERR_NOMEM : SFMB200_ERR_CUDA, \
                                "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));      \
    } while (0)

#define SFM_LAUNCH_CHECK(ctx)                                                                            \
    do {                                                                                                 \
        (ctx)->launches++;                                                                               \
        cudaError_t e_ = cudaGetLastError();                                                             \
        if (e_ != cudaSuccess)                                                                           \
            return sfmb200_fail((ctx), SFMB200_ERR_CUDA, "%s:%d kernel launch: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); \
    } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// multi-GPU (comm.cu): in-place sum over ranks of n doubles on the ctx stream; no-op when nranks == 1
int sfmb200_allreduce_sum_f64(sfmb200_ctx* ctx, double* dbuf, size_t n);
int sfmb200_allreduce_max_f64(sfmb200_ctx* ctx, double* dbuf, size_t n);
int sfmb200_allgather_bytes(sfmb200_ctx* ctx, const void* d_send, void* d_recv, size_t bytes);
void sfmb200_comm_destroy(sfmb200_ctx* ctx);

// image downscale (resize.cu), also run by the scaled JPEG decode (jpeg.cu) on the images it has just decoded.
// rz_plan: fills dw, dh, the tap offsets and the tiles of imgs[0..n) (sw, sh set by the caller) and appends their taps; false and the
// image in *bad if a size is refused.  rz_enqueue: one launch on ctx->stream over device copies of imgs / taps.
struct RzImg; struct RzTap;
bool rz_plan(double scale, RzImg* imgs, int n, std::vector<RzTap>& taps, int* bad);
int rz_enqueue(sfmb200_ctx* ctx, double scale, const RzImg* imgs, int n, const RzImg* d_imgs, const RzTap* d_taps, const uint8_t* d_src,
               uint8_t* d_dst);
