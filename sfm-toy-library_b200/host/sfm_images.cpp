// sfm_images.cpp -- sfmtoylib::readImages (sfm_images.h) over sfmb200_jpeg_info / sfmb200_decode_jpeg_batch, or with a downscale
// sfmb200_resize_size / sfmb200_decode_jpeg_batch_scaled; sfmtoylib::readImagesAndFeatures over sfmb200_decode_jpeg_extract_orb.
#include "sfm_images.h"
#include "../../include/sfmb200.h"
#include "sfm_features.h"

#include <algorithm>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <iterator>
#include <mutex>

namespace sfmtoylib {

namespace {

#if defined(SFMB200_WITH_OPENCV)
const int kType8UC3 = CV_8UC3;                // OpenCV's macro
#else
const int kType8UC3 = cv::CV_8UC3;            // cv_min.h
#endif

// one context per process (device from SFMB200_DEVICE, default 0), created on first use, like the stage shim's
sfmb200_ctx* context() {
    static sfmb200_ctx* ctx = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* dev = std::getenv("SFMB200_DEVICE");
        if (sfmb200_create(dev ? std::atoi(dev) : 0, &ctx) != SFMB200_OK) {
            std::cerr << "sfmb200: " << sfmb200_last_error(nullptr) << std::endl;
            ctx = nullptr;
        }
    });
    return ctx;
}

// The files of one call as bytes, and one output image per file sized as the decode (and downscale) will leave it.
struct Batch {
    std::vector<std::vector<uint8_t>> files;
    std::vector<const uint8_t*> data;
    std::vector<size_t> size;
    std::vector<cv::Mat> out;
    std::vector<uint8_t*> dst;
};

bool load(const std::vector<std::string>& filenames, double scale, float downscale, Batch& b) {
    const size_t n = filenames.size();
    b.files.resize(n); b.data.resize(n); b.size.resize(n); b.out.resize(n); b.dst.resize(n);
    for (size_t i = 0; i < n; ++i) {
        std::ifstream f(filenames[i], std::ios::binary);
        if (!f) { std::cerr << "Unable to read image from file: " << filenames[i] << std::endl; return false; }
        b.files[i].assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
        b.data[i] = b.files[i].data(); b.size[i] = b.files[i].size();
        int w = 0, h = 0, c = 0;
        if (sfmb200_jpeg_info(b.data[i], b.size[i], &w, &h, &c) != SFMB200_OK) {
            std::cerr << "Unable to read image from file: " << filenames[i] << " (not a JPEG file the GPU decoder supports)" << std::endl;
            return false;
        }
        if (scale != 1.0 && sfmb200_resize_size(w, h, scale, &w, &h) != SFMB200_OK) {
            std::cerr << "Unable to downscale image " << filenames[i] << " by " << downscale << std::endl;
            return false;
        }
        b.out[i] = cv::Mat(h, w, kType8UC3);
        b.dst[i] = b.out[i].data;
    }
    return true;
}

}  // namespace

bool readImages(const std::vector<std::string>& filenames, std::vector<cv::Mat>& images, float downscale) {
    const double scale = downscale;      // the reference's float factor, widened as cv::resize receives it
    Batch b;
    if (!load(filenames, scale, downscale, b)) return false;
    sfmb200_ctx* ctx = context();
    if (!ctx) return false;
    const int n = (int)b.files.size();
    const int rc = scale == 1.0 ? sfmb200_decode_jpeg_batch(ctx, b.data.data(), b.size.data(), n, b.dst.data(), nullptr)
                                : sfmb200_decode_jpeg_batch_scaled(ctx, b.data.data(), b.size.data(), n, scale, b.dst.data(), nullptr);
    if (rc != SFMB200_OK) {
        std::cerr << "sfmb200: decode_jpeg_batch: " << sfmb200_last_error(ctx) << std::endl;
        return false;
    }
    images.insert(images.end(), b.out.begin(), b.out.end());
    return true;
}

bool readImagesAndFeatures(const std::vector<std::string>& filenames, std::vector<cv::Mat>& images, std::vector<Features>& features,
                           float downscale) {
    const double scale = downscale;
    Batch b;
    if (!load(filenames, scale, downscale, b)) return false;
    sfmb200_ctx* ctx = context();
    if (!ctx) return false;
    const int n = (int)b.files.size(), nfeatures = 5000;                                 // ORB::create(5000), SfM2DFeatureUtilities.cpp:39
    int cap = nfeatures + 64;
    std::vector<sfmb200_keypoint> kp;
    std::vector<uint8_t> desc;
    std::vector<int32_t> cnt(n);
    for (;;) {
        kp.resize((size_t)n * cap); desc.resize((size_t)n * cap * 32);
        if (sfmb200_decode_jpeg_extract_orb(ctx, b.data.data(), b.size.data(), n, scale, nfeatures, cap, kp.data(), desc.data(), cnt.data(),
                                            b.dst.data(), nullptr) != SFMB200_OK) {
            std::cerr << "sfmb200: decode_jpeg_extract_orb: " << sfmb200_last_error(ctx) << std::endl;
            return false;
        }
        const int most = n ? *std::max_element(cnt.begin(), cnt.end()) : 0;
        if (most <= cap) break;
        cap = most;                                                                       // ties at a selection threshold: OpenCV keeps them all
    }
    images.insert(images.end(), b.out.begin(), b.out.end());
    for (int i = 0; i < n; ++i) features.push_back(featuresFromOrbRecords(kp.data() + (size_t)i * cap, desc.data() + (size_t)i * cap * 32, cnt[i]));
    return true;
}

}  // namespace sfmtoylib
