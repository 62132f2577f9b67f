// ctx.cu -- context lifetime and error reporting for libsfmb200.so (include/sfmb200.h).
#include "common.cuh"

static thread_local std::string g_create_error;

int sfmb200_fail(sfmb200_ctx* ctx, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (ctx) ctx->err = buf; else g_create_error = buf;
    return code;
}

int check_pair_batch(sfmb200_ctx* ctx, const float* pts, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs,
                     const int32_t* match_q, const int32_t* match_t, const int64_t* match_off, int64_t max_matches, int64_t* n_matches) {
    if (!img_off || (n_pairs > 0 && (!pairs || !match_off))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (img_off[0] != 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "img_off[0] must be 0");
    for (int i = 0; i < n_img; ++i)
        if (img_off[i + 1] < img_off[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "img_off is not monotone at image %d", i);
    if (img_off[n_img] > 0 && !pts) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (n_pairs > 0 && match_off[0] != 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_off[0] must be 0");
    for (int p = 0; p < n_pairs; ++p) {
        if (match_off[p + 1] < match_off[p]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_off is not monotone at pair %d", p);
        if (pairs[2 * p] < 0 || pairs[2 * p] >= n_img || pairs[2 * p + 1] < 0 || pairs[2 * p + 1] >= n_img)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair %d names an image outside [0, %d)", p, n_img);
    }
    const int64_t M = n_pairs > 0 ? match_off[n_pairs] : 0;
    if (M > max_matches) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "too many matches in one call");
    if (M > 0 && (!match_q || !match_t)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    for (int p = 0; p < n_pairs; ++p) {
        const int nl = img_off[pairs[2 * p] + 1] - img_off[pairs[2 * p]], nr = img_off[pairs[2 * p + 1] + 1] - img_off[pairs[2 * p + 1]];
        for (int64_t k = match_off[p]; k < match_off[p + 1]; ++k)
            if (match_q[k] < 0 || match_q[k] >= nl || match_t[k] < 0 || match_t[k] >= nr)
                return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match %lld of pair %d indexes outside its images' key points", (long long)k, p);
    }
    *n_matches = M;
    return SFMB200_OK;
}

int check_two_view_matches(sfmb200_ctx* ctx, const int32_t* match_q, const int32_t* match_t, int m, int n_left, int n_right) {
    if ((match_q == nullptr) != (match_t == nullptr)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_q and match_t must both be given or both be NULL");
    if (!match_q && (m > n_left || m > n_right)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "identity alignment needs m <= min(n_left, n_right)");
    if (match_q)
        for (int i = 0; i < m; ++i)
            if (match_q[i] < 0 || match_q[i] >= n_left || match_t[i] < 0 || match_t[i] >= n_right)
                return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match %d indexes outside the keypoint arrays", i);
    return SFMB200_OK;
}

extern "C" {

int sfmb200_version(void) { return SFMB200_VERSION; }

int sfmb200_create(int device, sfmb200_ctx** out) {
    if (!out) return SFMB200_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0)
        return sfmb200_fail(nullptr, SFMB200_ERR_CUDA, "no CUDA device available (%s); this library has no CPU fallback",
                            e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    if (device < 0 || device >= n) return sfmb200_fail(nullptr, SFMB200_ERR_INVALID, "device %d out of range [0,%d)", device, n);
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return sfmb200_fail(nullptr, SFMB200_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return sfmb200_fail(nullptr, SFMB200_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return sfmb200_fail(nullptr, SFMB200_ERR_UNSUPPORTED, "device %d is sm_%d%d; this build targets sm_90a (H100) only",
                            device, prop.major, prop.minor);
    sfmb200_ctx* c = new sfmb200_ctx();
    c->device = device; c->sm_count = prop.multiProcessorCount; c->l2_bytes = prop.l2CacheSize;
    e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { delete c; return sfmb200_fail(nullptr, SFMB200_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)); }
    *out = c;
    return SFMB200_OK;
}

void sfmb200_destroy(sfmb200_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto& e : ctx->ipc_cache) if (e.second) cudaIpcCloseMemHandle(e.second);
    ctx->ipc_cache.clear();
    sfmb200_comm_destroy(ctx);
    ctx->orb_dev.release(); ctx->orb_lists.release();
    ctx->orb_pin_img.release(); ctx->orb_pin_a.release(); ctx->orb_pin_b.release(); ctx->orb_pin_c.release(); ctx->orb_pin_tab.release();
    delete ctx->pool; ctx->pool = nullptr;
    if (ctx->orb_stream) cudaStreamDestroy(ctx->orb_stream);
    if (ctx->orb_up) cudaStreamDestroy(ctx->orb_up);
    for (auto& ev : ctx->orb_img_ev) if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->orb_ev) if (ev) cudaEventDestroy(ev);
    ctx->scratch.release(); ctx->scratch2.release(); ctx->pinned.release(); ctx->ba_ws.release(); ctx->mcache.release(); ctx->ds_ws.release();
    ctx->ess_trace.release();
    ctx->pose_trace.release();
    ctx->hg_trace.release();
    ctx->jpeg_dev.release(); ctx->jpeg_pin_up.release(); ctx->jpeg_pin_down.release();
    ctx->rz_dev.release(); ctx->rz_pin_up.release(); ctx->rz_pin_down.release();
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* sfmb200_last_error(const sfmb200_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }
void* sfmb200_stream(sfmb200_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int64_t sfmb200_kernel_launches(const sfmb200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int sfmb200_synchronize(sfmb200_ctx* ctx) {
    if (!ctx) return SFMB200_ERR_INVALID;
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SFMB200_OK;
}

}  // extern "C"
