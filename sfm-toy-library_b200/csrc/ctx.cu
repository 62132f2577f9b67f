// ctx.cu -- context lifetime and error reporting for libsfmb200.so (include/sfmb200.h).
#include "common.cuh"

static thread_local std::string g_create_error;

int sfmb200_fail(sfmb200_ctx* ctx, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (ctx) ctx->err = buf; else g_create_error = buf;
    return code;
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
    ctx->orb_pin_img.release(); ctx->orb_pin_a.release(); ctx->orb_pin_b.release(); ctx->orb_pin_c.release();
    delete ctx->pool; ctx->pool = nullptr;
    if (ctx->orb_stream) cudaStreamDestroy(ctx->orb_stream);
    if (ctx->orb_up) cudaStreamDestroy(ctx->orb_up);
    for (auto& ev : ctx->orb_img_ev) if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->orb_ev) if (ev) cudaEventDestroy(ev);
    ctx->scratch.release(); ctx->scratch2.release(); ctx->pinned.release(); ctx->ba_ws.release(); ctx->mcache.release(); ctx->ds_ws.release();
    ctx->ess_trace.release();
    ctx->hg_trace.release();
    ctx->jpeg_dev.release(); ctx->jpeg_pin_up.release(); ctx->jpeg_pin_down.release();
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
