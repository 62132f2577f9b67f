// decode.cu -- the host front end of the image decode entry points (include/sfmb200.h): sfmb200_decode_jpeg_batch[_scaled],
// sfmb200_decode_jpeg_extract_orb and sfmb200_decode_images[_extract_orb], and the host-only sfmb200_jpeg_info and sfmb200_image_info.
//
// Every check of a call passes before its first launch, in this order, each step over the files in the caller's order:
//   1. the arguments of the entry point
//   2. the format of every file: by signature for sfmb200_decode_images*, JPEG for the JPEG entry points
//   3. every file parsed once, on the host threads: the first file that does not parse or has no output buffer
//   4. the output sizes after the downscale: the first file the scale leaves with no pixels
//   5. per file: the output stride, then (ORB entry points) ORB's minimum and maximum image size
// Then the JPEG files run on jpeg.cu's backend and the PNG files on png.cu's, each into its own arena, so that both sets of images are
// alive on the device together when ORB takes them in the caller's order.
#include "common.cuh"
#include "png_parse.h"
#include "resize_math.cuh"

#include <cmath>

namespace {

// SFMB200_FORMAT_JPEG / _PNG by signature, 0 for neither
int image_format(const uint8_t* d, size_t n) {
    if (pg_is_png(d, n)) return SFMB200_FORMAT_PNG;
    if (d && n >= 2 && d[0] == 0xFF && d[1] == 0xD8) return SFMB200_FORMAT_JPEG;
    return 0;
}

// the parser of each format: the SFMB200 status, with the reason in `why`
int parse(const uint8_t* d, size_t n, JpImage& im, std::string& why) { return jp_parse(d, n, JD_CHUNK, im, why); }
int parse(const uint8_t* d, size_t n, PgImage& im, std::string& why) { return pg_parse(d, n, im, why); }

// the files of one format in a call: the caller's numbers and the parses
template <class Im> struct Files { std::vector<int> idx; std::vector<Im> ims; };

// Steps 1 (the checks every entry point shares) to 6.  mixed: sfmb200_decode_images*; orb: the images stay on the device for ORB
// (out_bgr may then be NULL).  On success call.dev, ow and oh describe the images on the device.
int decode(sfmb200_ctx* ctx, const char* name, bool mixed, bool orb, const size_t* size, int n, DecodeCall& call) {
    const uint8_t* const* data = call.data;
    // ---- 1. arguments
    if (n < 0 || (n > 0 && (!data || !size || (!call.out_bgr && !orb)))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: bad arguments", name);
    if (n > 65535) return sfmb200_fail(ctx, mixed ? SFMB200_ERR_UNSUPPORTED : SFMB200_ERR_INVALID, "%s: at most 65535 images per call", name);
    if (!std::isfinite(call.scale) || call.scale <= 0)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: scale %g is not a positive finite number", name, call.scale);
    for (int64_t& s : ctx->jpeg_stats) s = 0;
    if (mixed) for (int64_t& s : ctx->png_stats) s = 0;
    if (n == 0) return SFMB200_OK;

    // ---- 2. formats
    Files<JpImage> jpg;
    Files<PgImage> png;
    std::vector<int> slot(n);
    std::vector<char> is_png(n);
    for (int i = 0; i < n; ++i) {
        const int f = mixed ? image_format(data[i], size[i]) : SFMB200_FORMAT_JPEG;
        if (!f) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: neither a JPEG nor a PNG file", i);
        is_png[i] = f == SFMB200_FORMAT_PNG;
        std::vector<int>& idx = is_png[i] ? png.idx : jpg.idx;
        slot[i] = (int)idx.size();
        idx.push_back(i);
    }
    jpg.ims.resize(jpg.idx.size());
    png.ims.resize(png.idx.size());

    // ---- 3. parse
    std::vector<int> rc(n);
    std::vector<std::string> why(n);
    call.ow.resize(n); call.oh.resize(n);
    auto parse_one = [&](auto& files, int i) {
        auto& im = files.ims[slot[i]];
        rc[i] = parse(data[i], size[i], im, why[i]);
        call.ow[i] = im.OW; call.oh[i] = im.OH;
    };
    host_pool(ctx).parallel_for(n, [&](int i) { if (is_png[i]) parse_one(png, i); else parse_one(jpg, i); });
    for (int i = 0; i < n; ++i) {
        if (rc[i]) return sfmb200_fail(ctx, rc[i], "image %d: %s", i, why[i].c_str());
        if (call.out_bgr && !call.out_bgr[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: no output buffer", i);
    }

    // ---- 4. output sizes
    if (call.scale != 1.0)
        for (int i = 0; i < n; ++i) {
            const int w = call.ow[i], h = call.oh[i];
            if (!rz_size(w, h, call.scale, call.ow[i], call.oh[i]))
                return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: scale %g of a %dx%d image gives no image", i, call.scale, w, h);
        }

    // ---- 5. per file
    for (int i = 0; i < n; ++i) {
        const int ow = call.ow[i], oh = call.oh[i];
        if (call.out_bgr && call.out_stride && call.out_stride[i] && call.out_stride[i] < (size_t)ow * 3)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: output stride %zu < %d", i, call.out_stride[i], ow * 3);
        if (orb && (ow < 8 || oh < 8))
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: a %dx%d image is below ORB's minimum of 8 pixels per side", i, ow, oh);
        if (orb && (int64_t)ow * oh > ((int64_t)1 << 28))
            return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "image %d: a %dx%d image is too large for ORB (limit 2^28 pixels)", i, ow, oh);
    }

    // ---- 6. the backends
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    call.dev.resize(n);
    if (!jpg.idx.empty())
        if (int r = jd_run(ctx, call, jpg.idx, jpg.ims)) return r;
    if (!png.idx.empty())
        if (int r = pg_run(ctx, call, png.idx, png.ims)) return r;
    return SFMB200_OK;
}

// The decode into the caller's host buffers.
int decode_to_host(sfmb200_ctx* ctx, const char* name, bool mixed, const uint8_t* const* data, const size_t* size, int n, double scale,
                   uint8_t* const* out_bgr, const size_t* out_stride) {
    if (!ctx) return SFMB200_ERR_INVALID;
    DecodeCall call{data, scale, out_bgr, out_stride, {}, {}, {}};
    return decode(ctx, name, mixed, false, size, n, call);
}

// The decode with the images left on the device (and downloaded only with out_bgr), then one ORB pass over all of them.
int decode_extract_orb(sfmb200_ctx* ctx, const char* name, bool mixed, const uint8_t* const* data, const size_t* size, int n, double scale,
                       int nfeatures, int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints,
                       uint8_t* const* out_bgr, const size_t* out_stride) {
    if (!ctx) return SFMB200_ERR_INVALID;
    if (n < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: n < 0", name);
    if (n == 0) return SFMB200_OK;
    if (!keypoints || !descriptors || !n_keypoints || max_keypoints < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: null buffer", name);
    if (nfeatures < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "nfeatures < 0");
    std::lock_guard<std::mutex> lk(ctx->mu);
    DecodeCall call{data, scale, out_bgr, out_stride, {}, {}, {}};
    if (int rc = decode(ctx, name, mixed, true, size, n, call)) return rc;
    return orb_extract_device(ctx, call.dev.data(), call.ow.data(), call.oh.data(), n, nfeatures, max_keypoints, keypoints, descriptors, n_keypoints);
}

}  // namespace

extern "C" {

int sfmb200_jpeg_info(const uint8_t* data, size_t size, int* width, int* height, int* components) {
    JpImage im;
    std::string why;
    if (int rc = parse(data, size, im, why)) return rc;
    if (width) *width = im.OW;
    if (height) *height = im.OH;
    if (components) *components = im.ncomp;
    return SFMB200_OK;
}

int sfmb200_image_info(const uint8_t* data, size_t size, int* format, int* width, int* height) {
    // a refusal leaves its reason in sfmb200_last_error(NULL)
    const int f = image_format(data, size);
    if (!f) return sfmb200_fail(nullptr, SFMB200_ERR_INVALID, "neither a JPEG nor a PNG file");
    JpImage jp;
    PgImage pg;
    std::string why;
    if (int rc = f == SFMB200_FORMAT_PNG ? parse(data, size, pg, why) : parse(data, size, jp, why)) return sfmb200_fail(nullptr, rc, "%s", why.c_str());
    if (format) *format = f;
    if (width) *width = f == SFMB200_FORMAT_PNG ? pg.OW : jp.OW;
    if (height) *height = f == SFMB200_FORMAT_PNG ? pg.OH : jp.OH;
    return SFMB200_OK;
}

int sfmb200_decode_jpeg_batch(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, uint8_t* const* out_bgr,
                              const size_t* out_stride) {
    return decode_to_host(ctx, "decode_jpeg_batch", false, data, size, n, 1.0, out_bgr, out_stride);
}

int sfmb200_decode_jpeg_batch_scaled(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale,
                                     uint8_t* const* out_bgr, const size_t* out_stride) {
    return decode_to_host(ctx, "decode_jpeg_batch_scaled", false, data, size, n, scale, out_bgr, out_stride);
}

int sfmb200_decode_jpeg_extract_orb(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, int nfeatures,
                                    int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints,
                                    uint8_t* const* out_bgr, const size_t* out_stride) {
    return decode_extract_orb(ctx, "decode_jpeg_extract_orb", false, data, size, n, scale, nfeatures, max_keypoints, keypoints, descriptors,
                              n_keypoints, out_bgr, out_stride);
}

int sfmb200_decode_images(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, uint8_t* const* out_bgr,
                          const size_t* out_stride) {
    if (ctx && n > 0 && !out_bgr) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "decode_images: no output buffers");
    return decode_to_host(ctx, "decode_images", true, data, size, n, scale, out_bgr, out_stride);
}

int sfmb200_decode_images_extract_orb(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, int nfeatures,
                                      int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints,
                                      uint8_t* const* out_bgr, const size_t* out_stride) {
    return decode_extract_orb(ctx, "decode_images_extract_orb", true, data, size, n, scale, nfeatures, max_keypoints, keypoints, descriptors,
                              n_keypoints, out_bgr, out_stride);
}

}  // extern "C"
