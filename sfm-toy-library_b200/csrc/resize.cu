// resize.cu -- the downscale of SfM::setImagesDirectory (cv::resize(img, img, Size(), s, s), INTER_LINEAR) for a batch of 8-bit
// B,G,R images on the device, byte-identical to OpenCV 4.13 (include/sfmb200.h; the arithmetic is csrc/resize_math.cuh).
//
// One launch covers every image of a call, the image index in blockIdx.y (like jd_color):
//   rz_linear   one CTA per RZ_TW x RZ_TH output tile: the horizontal pass of the two source rows of every output row of the tile into
//               shared memory (int32), then the vertical pass, packed B,G,R out
//   rz_area     1 / s == 2: one thread per output pixel, the 2x2 block average with its edge rule
// The taps are built on the host (rz_plan) and ride in the call's one upload.  The scaled decodes (jpeg.cu, png.cu) run the same kernels
// on the images they have just decoded.
#include "common.cuh"
#include "resize_math.cuh"

#include <cmath>

namespace {

constexpr int RZ_TW = 64, RZ_TH = 4, RZ_THREADS = RZ_TW * RZ_TH;

__global__ void __launch_bounds__(RZ_THREADS) rz_linear(const RzImg* __restrict__ imgs, const RzTap* __restrict__ taps,
                                                        const uint8_t* __restrict__ src, uint8_t* __restrict__ dst) {
    __shared__ int32_t hb[2 * RZ_TH][3 * RZ_TW];
    const RzImg& im = imgs[blockIdx.y];
    if ((int)blockIdx.x >= im.ntiles) return;
    const int x0 = (blockIdx.x % im.tiles_x) * RZ_TW, y0 = (blockIdx.x / im.tiles_x) * RZ_TH;
    const uint8_t* s = src + im.src0;
    for (int k = threadIdx.x; k < 2 * RZ_TH * RZ_TW; k += RZ_THREADS) {
        const int r = k / RZ_TW, x = k % RZ_TW, dx = x0 + x, dy = y0 + r / 2;
        if (dx >= im.dw || dy >= im.dh) continue;
        const RzTap ty = taps[im.tap_y + dy], tx = taps[im.tap_x + dx];
        const uint8_t* row = s + (long long)(r & 1 ? ty.i1 : ty.i0) * im.src_stride;
        for (int c = 0; c < 3; ++c) hb[r][3 * x + c] = rz_hpass(row, tx, c);
    }
    __syncthreads();
    const int x = threadIdx.x % RZ_TW, r = threadIdx.x / RZ_TW, dx = x0 + x, dy = y0 + r;
    if (dx >= im.dw || dy >= im.dh) return;
    const RzTap ty = taps[im.tap_y + dy];
    uint8_t* o = dst + im.dst0 + dy * im.dst_stride + 3 * dx;
    for (int c = 0; c < 3; ++c) o[c] = rz_vpass(hb[2 * r][3 * x + c], hb[2 * r + 1][3 * x + c], ty.a0, ty.a1);
}

__global__ void __launch_bounds__(256) rz_area(const RzImg* __restrict__ imgs, const uint8_t* __restrict__ src, uint8_t* __restrict__ dst) {
    const RzImg& im = imgs[blockIdx.y];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (long long)im.dw * im.dh) return;
    const int dx = (int)(p % im.dw), dy = (int)(p / im.dw);
    uint8_t* o = dst + im.dst0 + dy * im.dst_stride + 3 * dx;
    for (int c = 0; c < 3; ++c) o[c] = rz_area2(src + im.src0, im.src_stride, im.sw, im.sh, dx, dy, c);
}

}  // namespace

bool rz_plan(double scale, RzImg* imgs, int n, std::vector<RzTap>& taps, int* bad) {
    for (int i = 0; i < n; ++i) {
        RzImg& d = imgs[i];
        if (!rz_size(d.sw, d.sh, scale, d.dw, d.dh)) { if (bad) *bad = i; return false; }
        d.tap_x = (int)taps.size(); d.tap_y = d.tap_x + d.dw;
        taps.resize(taps.size() + d.dw + d.dh);
        rz_taps(d.sw, d.sh, d.dw, d.dh, scale, taps.data() + d.tap_x, taps.data() + d.tap_y);
        d.tiles_x = ceil_div(d.dw, RZ_TW);
        d.ntiles = (int)std::min<long long>(INT32_MAX, (long long)d.tiles_x * ceil_div(d.dh, RZ_TH));
    }
    return true;
}

int rz_enqueue(sfmb200_ctx* ctx, double scale, const RzImg* imgs, int n, const RzImg* d_imgs, const RzTap* d_taps, const uint8_t* d_src,
               uint8_t* d_dst) {
    if (n <= 0) return SFMB200_OK;
    if (rz_is_area2(scale)) {
        long long max_pix = 0;
        for (int i = 0; i < n; ++i) max_pix = std::max(max_pix, (long long)imgs[i].dw * imgs[i].dh);
        rz_area<<<dim3((unsigned)ceil_div64(max_pix, 256), (unsigned)n), 256, 0, ctx->stream>>>(d_imgs, d_src, d_dst);
    } else {
        int max_tiles = 0;
        for (int i = 0; i < n; ++i) max_tiles = std::max(max_tiles, imgs[i].ntiles);
        rz_linear<<<dim3((unsigned)max_tiles, (unsigned)n), RZ_THREADS, 0, ctx->stream>>>(d_imgs, d_taps, d_src, d_dst);
    }
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

extern "C" {

int sfmb200_resize_size(int w, int h, double scale, int* dw, int* dh) {
    int a = 0, b = 0;
    if (!rz_size(w, h, scale, a, b)) return SFMB200_ERR_INVALID;
    if (dw) *dw = a;
    if (dh) *dh = b;
    return SFMB200_OK;
}

int sfmb200_resize_batch(sfmb200_ctx* ctx, const uint8_t* const* src, const int* w, const int* h, const size_t* src_stride, int n,
                         double scale, uint8_t* const* dst, const size_t* dst_stride) {
    if (!ctx) return SFMB200_ERR_INVALID;
    if (n < 0 || (n > 0 && (!src || !w || !h || !dst))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "resize_batch: bad arguments");
    if (n > 65535) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "resize_batch: at most 65535 images per call");
    if (!std::isfinite(scale) || scale <= 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "resize_batch: scale %g is not a positive finite number", scale);
    std::vector<RzImg> img(n);
    for (int i = 0; i < n; ++i) {
        memset(&img[i], 0, sizeof(RzImg));
        img[i].sw = w[i]; img[i].sh = h[i];
        if (!src[i] || !dst[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: no buffer", i);
        if (w[i] <= 0 || h[i] <= 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: size %dx%d", i, w[i], h[i]);
        if (src_stride && src_stride[i] && src_stride[i] < (size_t)w[i] * 3)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: source stride %zu < %d", i, src_stride[i], w[i] * 3);
    }
    std::vector<RzTap> taps;
    int bad = 0;
    if (!rz_plan(scale, img.data(), n, taps, &bad))
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: scale %g of a %dx%d image gives no image", bad, scale, w[bad], h[bad]);
    for (int i = 0; i < n; ++i)
        if (dst_stride && dst_stride[i] && dst_stride[i] < (size_t)img[i].dw * 3)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: output stride %zu < %d", i, dst_stride[i], img[i].dw * 3);
    if (n == 0) return SFMB200_OK;
    HostPool& pool = host_pool(ctx);
    auto srow = [&](int i) { return src_stride && src_stride[i] ? src_stride[i] : (size_t)w[i] * 3; };
    auto drow = [&](int i) { return dst_stride && dst_stride[i] ? dst_stride[i] : (size_t)img[i].dw * 3; };
    if (scale == 1.0) {                 // SfM::setImagesDirectory does not call cv::resize for a factor of 1: the input bytes
        pool.parallel_for(n, [&](int i) { copy_rows(dst[i], drow(i), src[i], srow(i), (size_t)w[i] * 3, h[i]); });
        return SFMB200_OK;
    }
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));

    // ---- layout: descriptors, taps and packed source images up; packed resized images down
    long long inb = 0, outb = 0;
    for (int i = 0; i < n; ++i) {
        RzImg& d = img[i];
        d.src0 = inb; d.src_stride = (long long)d.sw * 3; inb += (long long)al256((size_t)d.src_stride * d.sh);
        d.dst0 = outb; d.dst_stride = (long long)d.dw * 3; outb += (long long)al256((size_t)d.dst_stride * d.dh);
    }
    const size_t o_img = 0, o_tap = al256(sizeof(RzImg) * n), o_src = o_tap + al256(sizeof(RzTap) * taps.size());
    const size_t up_bytes = o_src + (size_t)inb, o_dst = al256(up_bytes), total = o_dst + (size_t)outb;
    SFM_CUDA(ctx, ctx->rz_pin_up.reserve(up_bytes));
    SFM_CUDA(ctx, ctx->rz_pin_down.reserve((size_t)outb));
    SFM_CUDA(ctx, ctx->rz_dev.reserve(total));
    char* up = (char*)ctx->rz_pin_up.p;
    memcpy(up + o_img, img.data(), sizeof(RzImg) * n);
    memcpy(up + o_tap, taps.data(), sizeof(RzTap) * taps.size());
    pool.parallel_for(n, [&](int i) {
        const size_t row = (size_t)img[i].src_stride;
        copy_rows((uint8_t*)up + o_src + img[i].src0, row, src[i], srow(i), row, img[i].sh);
    });
    char* dv = (char*)ctx->rz_dev.p;
    cudaStream_t st = ctx->stream;
    SFM_CUDA(ctx, cudaMemcpyAsync(dv, up, up_bytes, cudaMemcpyHostToDevice, st));
    if (int rc = rz_enqueue(ctx, scale, img.data(), n, (const RzImg*)(dv + o_img), (const RzTap*)(dv + o_tap), (const uint8_t*)(dv + o_src),
                            (uint8_t*)(dv + o_dst)))
        return rc;
    char* hd = (char*)ctx->rz_pin_down.p;
    SFM_CUDA(ctx, cudaMemcpyAsync(hd, dv + o_dst, (size_t)outb, cudaMemcpyDeviceToHost, st));
    SFM_CUDA(ctx, cudaStreamSynchronize(st));
    pool.parallel_for(n, [&](int i) {
        const size_t row = (size_t)img[i].dst_stride;
        copy_rows(dst[i], drow(i), (const uint8_t*)hd + img[i].dst0, row, row, img[i].dh);
    });
    return SFMB200_OK;
}

}  // extern "C"
