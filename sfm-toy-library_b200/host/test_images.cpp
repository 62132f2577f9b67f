// test_images.cpp -- drives sfmtoylib::readImages (sfm_images.h) for tests/test_gpu_host_shim_images.py, which compares its output
// with cv2.imdecode.  Usage: test_images <out.bin> <file.jpg>...
// out.bin (little endian): per image int32 rows, cols, then rows * cols * 3 bytes (B,G,R).
#include "sfm_images.h"
#include <cstdio>

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    std::vector<std::string> names(argv + 2, argv + argc);
    std::vector<cv::Mat> images;
    if (!sfmtoylib::readImages(names, images)) { std::printf("IMAGES_TEST FAIL (readImages)\n"); return 1; }
    FILE* f = std::fopen(argv[1], "wb");
    if (!f) return 2;
    for (const cv::Mat& m : images) {
        const int32_t hw[2] = {m.rows, m.cols};
        std::fwrite(hw, sizeof hw, 1, f);
        std::fwrite(m.data, 1, (size_t)m.rows * m.cols * 3, f);
    }
    std::fclose(f);
    std::printf("IMAGES_TEST PASS (%zu images)\n", images.size());
    return 0;
}
