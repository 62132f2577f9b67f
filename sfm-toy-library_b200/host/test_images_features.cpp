// test_images_features.cpp -- drives sfmtoylib::readImagesAndFeatures (sfm_images.h) for tests/test_gpu_host_images_features.py, which
// compares its output with the Python stage.  Usage: test_images_features [-s <scale>] <out.bin> <file.jpg>...
// out.bin (little endian): per image int32 rows, cols, then rows * cols * 3 bytes (B,G,R); int32 n, n key points (28 bytes each,
// cv::KeyPoint), n * 32 descriptor bytes, n points (2 float32 each).
#include "sfm_images.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>

int main(int argc, char** argv) {
    float downscale = 1.0f;
    if (argc >= 3 && std::strcmp(argv[1], "-s") == 0) {
        downscale = std::strtof(argv[2], nullptr);
        argc -= 2; argv += 2;
    }
    if (argc < 3) return 2;
    std::vector<std::string> names(argv + 2, argv + argc);
    std::vector<cv::Mat> images;
    std::vector<sfmtoylib::Features> features;
    if (!sfmtoylib::readImagesAndFeatures(names, images, features, downscale)) { std::printf("IMAGES_FEATURES_TEST FAIL\n"); return 1; }
    if (images.size() != names.size() || features.size() != names.size()) { std::printf("IMAGES_FEATURES_TEST FAIL (counts)\n"); return 1; }
    FILE* f = std::fopen(argv[1], "wb");
    if (!f) return 2;
    for (size_t i = 0; i < images.size(); ++i) {
        const cv::Mat& m = images[i];
        const int32_t hw[2] = {m.rows, m.cols};
        std::fwrite(hw, sizeof hw, 1, f);
        std::fwrite(m.data, 1, (size_t)m.rows * m.cols * 3, f);
        const sfmtoylib::Features& ft = features[i];
        const int32_t n = (int32_t)ft.keyPoints.size();
        std::fwrite(&n, 4, 1, f);
        std::fwrite(ft.keyPoints.data(), sizeof(cv::KeyPoint), n, f);
        if (n) std::fwrite(ft.descriptors.data, 1, 32 * (size_t)n, f);
        std::fwrite(ft.points.data(), sizeof(cv::Point2f), ft.points.size(), f);
    }
    std::fclose(f);
    std::printf("IMAGES_FEATURES_TEST PASS (%zu images)\n", images.size());
    return 0;
}
