// test_shim_homography.cpp -- C++ host-side test of the shim built with SFMB200_SHIM_HOMOGRAPHY (runs on the GPU box):
// findHomographyInliers on a planar pair with a known homography, 150 exact inliers and 50 far outliers, counts the inliers.
#include "sfmtoylib_b200.h"

#include <cstdio>
#include <random>

using namespace sfmtoylib;

static int failures = 0;
#define EXPECT(cond, msg) do { if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } } while (0)

int main() {
    const double H[9] = {0.97, 0.03, 25.0, -0.02, 1.04, -8.0, 1e-5, 2e-5, 1.0};
    std::mt19937 rng(11);
    std::uniform_real_distribution<double> ux(0, 1024), uy(0, 768), off(150, 300);
    Features left, right; Matching matching;
    for (int i = 0; i < 200; ++i) {
        const double x = ux(rng), y = uy(rng), w = H[6] * x + H[7] * y + H[8];
        double u = (H[0] * x + H[1] * y + H[2]) / w, v = (H[3] * x + H[4] * y + H[5]) / w;
        if (i >= 150) { u += (i & 1 ? 1 : -1) * off(rng); v += (i & 2 ? 1 : -1) * off(rng); }
        left.points.push_back(cv::Point2f((float)x, (float)y));
        right.points.push_back(cv::Point2f((float)u, (float)v));
        matching.push_back(cv::DMatch(i, i, 0));
    }
    const int n = SfMStereoUtilities::findHomographyInliers(left, right, matching);
    EXPECT(n == 150, "the 150 planted inliers are counted");
    Matching few(matching.begin(), matching.begin() + 3);
    EXPECT(SfMStereoUtilities::findHomographyInliers(left, right, few) == 0, "three matches: 0");
    std::printf("inliers %d of %zu\n", n, matching.size());
    std::printf(failures ? "SHIM_HOMOGRAPHY_TEST FAIL (%d)\n" : "SHIM_HOMOGRAPHY_TEST PASS\n", failures);
    return failures ? 1 : 0;
}
