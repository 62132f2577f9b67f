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
#include "match_cache.h"

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

// bytes rounded up to the 256-byte alignment of every buffer carved out of a DevBuf / PinBuf
static inline size_t al256(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// bump allocator over a DevBuf: carve() after a single reserve()
struct Carver {
    char* base; size_t off = 0;
    explicit Carver(void* b) : base((char*)b) {}
    template <typename T> T* take(size_t n) {
        off = al256(off);
        T* r = (T*)(base + off); off += n * sizeof(T); return r;
    }
    static size_t pad(size_t bytes) { return al256(bytes); }
};

// h rows of `row` bytes from src (rows src_stride bytes apart) to dst (rows dst_stride bytes apart): one memcpy when both are packed.
static inline void copy_rows(uint8_t* dst, size_t dst_stride, const uint8_t* src, size_t src_stride, size_t row, int h) {
    if (dst_stride == row && src_stride == row) memcpy(dst, src, row * h);
    else for (int y = 0; y < h; ++y) memcpy(dst + y * dst_stride, src + y * src_stride, row);
}

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
// expanded tensor-core operand blocks, bump-allocated, flushed whole when full (bookkeeping and capacity plan: match_cache.h).
struct MatchCache : MatchCacheState {
    DevBuf desc, exp;
    void release() { desc.release(); exp.release(); reset(); }
};

// Device buffers of the last ORB extraction group (orb.cu), kept for sfmb200_orb_download_level (stage-by-stage parity tests): the
// size of each of its images and where that image's pyramid starts in the three arenas.
struct OrbLast {
    uint8_t *pyr = nullptr, *blur = nullptr, *score = nullptr; int nimg = 0, nfeatures = 0;
    std::vector<int> w, h; std::vector<size_t> pix0;
};

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
    PinBuf orb_pin_tab;         // ORB extraction: a group's layouts, resize taps and tile lists, staged for their one upload
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
    DevBuf pose_trace;          // samples / inlier counts of the last PnP RANSAC (pose.cu)
    int pose_trace_samples = 0;
    DevBuf hg_trace;            // visited samples / counts of the last homography RANSAC with record_trace (homography.cu)
    int hg_trace_pairs = 0, hg_trace_stride = 0;
    std::vector<int32_t> hg_trace_visited;
    DevBuf jpeg_dev;                    // JPEG decoding (jpeg.cu): tables, entropy data, coefficients, planes, images of the last batch
    PinBuf jpeg_pin_up, jpeg_pin_down;  // its one upload and its one download
    int64_t jpeg_stats[7] = {0, 0, 0, 0, 0, 0, 0};   // sfmb200_jpeg_last_stats of the last batch
    DevBuf png_dev;                     // PNG decoding (png.cu): the images of the last call, then one group's IDAT data and work arrays
    PinBuf png_pin_up, png_pin_down;    // a group's one upload and its one download
    int64_t png_stats[SFMB200_PNG_STATS] = {};       // sfmb200_png_last_stats of the last call
    DevBuf rz_dev;                      // image downscale (resize.cu): descriptors, taps, source and resized images of the last batch
    PinBuf rz_pin_up, rz_pin_down;      // its one upload and its one download
};

int sfmb200_fail(sfmb200_ctx* ctx, int code, const char* fmt, ...);

// the context's host threads, created on first use
static inline HostPool& host_pool(sfmb200_ctx* ctx) {
    if (!ctx->pool) ctx->pool = new HostPool(HostPool::default_threads() - 1);
    return *ctx->pool;
}

// Host-side input checks shared by several entry points (ctx.cu).  Each returns SFMB200_OK, or SFMB200_ERR_INVALID with the
// message set through sfmb200_fail.
// check_pair_batch: the image-pair batch layout of include/sfmb200.h (pts / img_off / pairs / match_q / match_t / match_off) with
// at most max_matches matches; on success *n_matches = match_off[n_pairs], or 0 when n_pairs == 0.
int check_pair_batch(sfmb200_ctx* ctx, const float* pts, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs,
                     const int32_t* match_q, const int32_t* match_t, const int64_t* match_off, int64_t max_matches, int64_t* n_matches);
// check_two_view_matches: match_q / match_t [m] of a single-pair call index pts_left [n_left] / pts_right [n_right]; both NULL
// means identity alignment, which needs m <= min(n_left, n_right).
int check_two_view_matches(sfmb200_ctx* ctx, const int32_t* match_q, const int32_t* match_t, int m, int n_left, int n_right);

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
// ORB extraction of images already on the device (orb.cu): packed B,G,R rows of ws[i] x hs[i] pixels at d_bgr[i], any sizes; results as
// sfmb200_orb_detect_and_compute_batch.  The caller holds ctx->mu and has checked the sizes.
int orb_extract_device(sfmb200_ctx* ctx, const uint8_t* const* d_bgr, const int* ws, const int* hs, int n, int nfeatures, int max_keypoints,
                       sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints);

struct RzImg; struct RzTap;
bool rz_plan(double scale, RzImg* imgs, int n, std::vector<RzTap>& taps, int* bad);
int rz_enqueue(sfmb200_ctx* ctx, double scale, const RzImg* imgs, int n, const RzImg* d_imgs, const RzTap* d_taps, const uint8_t* d_src,
               uint8_t* d_dst);

// image decoding: decode.cu checks a call and parses its files, then the JPEG (jpeg.cu) and PNG (png.cu) backends run them.
constexpr int JD_CHUNK = 4096;        // bytes per unstuffing CTA of jpeg.cu, the unit jp_parse counts dropped bytes in

// A decode call that has passed every check: the caller's arrays, indexed by the caller's image numbers, and every image's output size
// (after the downscale).  The backend of image i sets dev[i] to where the image stays on the device, packed B,G,R rows, until the next
// decode of its format.  out_bgr NULL: the images are not downloaded.
struct DecodeCall {
    const uint8_t* const* data;
    double scale;
    uint8_t* const* out_bgr;
    const size_t* out_stride;
    std::vector<int> ow, oh;
    std::vector<const uint8_t*> dev;
    size_t stride(int i) const { return out_stride && out_stride[i] ? out_stride[i] : (size_t)ow[i] * 3; }
};
// The call's files idx[k], parsed into ims[k].  Each backend refuses only what its device layout cannot hold, before its first launch,
// and what its kernels find.
struct JpImage; struct PgImage;
int jd_run(sfmb200_ctx* ctx, DecodeCall& call, const std::vector<int>& idx, const std::vector<JpImage>& ims);
int pg_run(sfmb200_ctx* ctx, DecodeCall& call, const std::vector<int>& idx, const std::vector<PgImage>& ims);
