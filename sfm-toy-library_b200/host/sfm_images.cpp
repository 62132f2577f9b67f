// sfm_images.cpp -- sfmtoylib::readImages (sfm_images.h) over sfmb200_jpeg_info / sfmb200_decode_jpeg_batch, or with a downscale
// sfmb200_resize_size / sfmb200_decode_jpeg_batch_scaled.
#include "sfm_images.h"
#include "../../include/sfmb200.h"

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

}  // namespace

bool readImages(const std::vector<std::string>& filenames, std::vector<cv::Mat>& images, float downscale) {
    const double scale = downscale;      // the reference's float factor, widened as cv::resize receives it
    std::vector<std::vector<uint8_t>> files(filenames.size());
    std::vector<const uint8_t*> data(files.size());
    std::vector<size_t> size(files.size());
    std::vector<cv::Mat> out(files.size());
    std::vector<uint8_t*> dst(files.size());
    for (size_t i = 0; i < files.size(); ++i) {
        std::ifstream f(filenames[i], std::ios::binary);
        if (!f) { std::cerr << "Unable to read image from file: " << filenames[i] << std::endl; return false; }
        files[i].assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
        data[i] = files[i].data(); size[i] = files[i].size();
        int w = 0, h = 0, c = 0;
        if (sfmb200_jpeg_info(data[i], size[i], &w, &h, &c) != SFMB200_OK) {
            std::cerr << "Unable to read image from file: " << filenames[i] << " (not a JPEG file the GPU decoder supports)" << std::endl;
            return false;
        }
        if (scale != 1.0 && sfmb200_resize_size(w, h, scale, &w, &h) != SFMB200_OK) {
            std::cerr << "Unable to downscale image " << filenames[i] << " by " << downscale << std::endl;
            return false;
        }
        out[i] = cv::Mat(h, w, kType8UC3);
        dst[i] = out[i].data;
    }
    sfmb200_ctx* ctx = context();
    if (!ctx) return false;
    const int rc = scale == 1.0 ? sfmb200_decode_jpeg_batch(ctx, data.data(), size.data(), (int)files.size(), dst.data(), nullptr)
                                : sfmb200_decode_jpeg_batch_scaled(ctx, data.data(), size.data(), (int)files.size(), scale, dst.data(), nullptr);
    if (rc != SFMB200_OK) {
        std::cerr << "sfmb200: decode_jpeg_batch: " << sfmb200_last_error(ctx) << std::endl;
        return false;
    }
    images.insert(images.end(), out.begin(), out.end());
    return true;
}

}  // namespace sfmtoylib
