// test_shim_essential.cpp -- C++ host-side test of the shim built with SFMB200_SHIM_ESSENTIAL (runs on the GPU box):
// findCameraMatricesFromMatch on the reference's triangulate_from_2_views stereo scene (SfMUnitTests.cpp: 12 canned points,
// two mock cameras) recovers the relative pose of the two cameras.
#include "sfmtoylib_b200.h"

#include <cmath>
#include <cstdio>

using namespace sfmtoylib;

static int failures = 0;
#define EXPECT(cond, msg) do { if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } } while (0)

static void eulerDegToR(double pitch, double roll, double yaw, double R[9]) {      // R = Rz(yaw) Ry(roll) Rx(pitch)
    const double d = M_PI / 180.0, c1 = std::cos(yaw * d), s1 = std::sin(yaw * d), c2 = std::cos(roll * d), s2 = std::sin(roll * d),
                 c3 = std::cos(pitch * d), s3 = std::sin(pitch * d);
    const double r[9] = {c1 * c2, -s1 * c3 + c1 * s2 * s3, s1 * s3 + c1 * s2 * c3, s1 * c2, c1 * c3 + s1 * s2 * s3, -c1 * s3 + s1 * s2 * c3, -s2, c2 * s3, c2 * c3};
    for (int i = 0; i < 9; ++i) R[i] = r[i];
}

int main() {
    const double canned[12][3] = {{4, 12, 50}, {12, 11, 55}, {22, 1, 45}, {13, 3, 60}, {11, 16, 61}, {21, 12, 65}, {24, 11, 67},
                                  {29, 6, 41}, {27, 4, 44}, {22, 7, 58}, {20, 9, 51}, {15, 10, 40}};
    double Rl[9], Rr[9];
    eulerDegToR(5, 5, 5, Rl); eulerDegToR(-5, 0, 5, Rr);
    const double tl[3] = {-10, 0, 30}, tr[3] = {10, 0, 28}, f = 700, cx = 320, cy = 240;
    Features left, right; Matching matching;
    for (int i = 0; i < 12; ++i) {
        double pl[3], pr[3];
        for (int r = 0; r < 3; ++r) {
            pl[r] = Rl[3 * r] * canned[i][0] + Rl[3 * r + 1] * canned[i][1] + Rl[3 * r + 2] * canned[i][2] + tl[r];
            pr[r] = Rr[3 * r] * canned[i][0] + Rr[3 * r + 1] * canned[i][1] + Rr[3 * r + 2] * canned[i][2] + tr[r];
        }
        left.points.push_back(cv::Point2f((float)(f * pl[0] / pl[2] + cx), (float)(f * pl[1] / pl[2] + cy)));
        right.points.push_back(cv::Point2f((float)(f * pr[0] / pr[2] + cx), (float)(f * pr[1] / pr[2] + cy)));
        matching.push_back(cv::DMatch(i, i, 0));
    }
    Intrinsics intr; intr.K = cv::Mat(3, 3, cv::CV_32F);
    const float k[9] = {700, 0, 320, 0, 700, 240, 0, 0, 1};
    for (int i = 0; i < 9; ++i) intr.K.ptr<float>(0)[i] = k[i];
    // relative pose of the right camera in the left camera's frame: R = Rr Rl^T, t = tr - R tl (up to scale)
    double R[9], t[3], tn = 0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[3 * i + j] = Rr[3 * i] * Rl[3 * j] + Rr[3 * i + 1] * Rl[3 * j + 1] + Rr[3 * i + 2] * Rl[3 * j + 2];
    for (int i = 0; i < 3; ++i) { t[i] = tr[i] - (R[3 * i] * tl[0] + R[3 * i + 1] * tl[1] + R[3 * i + 2] * tl[2]); tn += t[i] * t[i]; }
    tn = std::sqrt(tn);
    Matching pruned; cv::Matx34f Pl, Pr;
    const bool ok = SfMStereoUtilities::findCameraMatricesFromMatch(intr, matching, left, right, pruned, Pl, Pr);
    EXPECT(ok, "a pose is found");
    EXPECT(pruned.size() == 12, "all 12 matches kept");
    double dr = 0, dt = 0;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) dr = std::fmax(dr, std::fabs(Pr(i, j) - R[3 * i + j]));
        dt = std::fmax(dt, std::fabs(Pr(i, 3) - t[i] / tn));
    }
    EXPECT(dr < 1e-3, "rotation within 1e-3");
    EXPECT(dt < 1e-2, "translation direction within 1e-2");
    EXPECT(Pl(0, 0) == 1 && Pl(1, 1) == 1 && Pl(2, 2) == 1 && Pl(0, 3) == 0, "Pleft = [I|0]");
    Matching few(matching.begin(), matching.begin() + 4);
    EXPECT(!SfMStereoUtilities::findCameraMatricesFromMatch(intr, few, left, right, pruned, Pl, Pr), "four matches: no model");
    std::printf("rotation error %.3g, translation error %.3g\n", dr, dt);
    std::printf(failures ? "SHIM_ESSENTIAL_TEST FAIL (%d)\n" : "SHIM_ESSENTIAL_TEST PASS\n", failures);
    return failures ? 1 : 0;
}
