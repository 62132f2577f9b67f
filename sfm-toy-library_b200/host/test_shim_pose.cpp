// test_shim_pose.cpp -- C++ host-side test of the shim built with SFMB200_SHIM_POSE (runs on the GPU box).
// Without arguments: findCameraPoseFrom2D3DMatch on the reference's find_camera_pose_from_2d3d_match scene (SfMUnitTests.cpp: 12
// canned points seen by a mock camera) recovers the camera to the reference's tolerances, and a set whose correspondences are
// scrambled fails the ratio test without touching the pose.
// With a file argument (int32 m, float K[9], float points3D[m][3], float points2D[m][2]): prints the decision and the pose as
// hexadecimal floats, for the Python test to compare with ransac.findCameraPoseFrom2D3DMatch_gpu.
#include "sfm_glue.h"

#include <cmath>
#include <cstdio>

using namespace sfmtoylib;

static int failures = 0;
#define EXPECT(cond, msg) do { if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } } while (0)

static Intrinsics intrinsics(const float* k) {
    Intrinsics intr; intr.K = cv::Mat(3, 3, cv::CV_32F);
    for (int i = 0; i < 9; ++i) intr.K.ptr<float>(0)[i] = k[i];
    return intr;
}

static int from_file(const char* path) {
    FILE* f = std::fopen(path, "rb");
    if (!f) { std::printf("cannot open %s\n", path); return 2; }
    int32_t m = 0; float k[9];
    bool ok = std::fread(&m, 4, 1, f) == 1 && std::fread(k, 4, 9, f) == 9;
    Image2D3DMatch match;
    match.points3D.resize(ok ? m : 0); match.points2D.resize(ok ? m : 0);
    ok = ok && std::fread(match.points3D.data(), 12, m, f) == (size_t)m && std::fread(match.points2D.data(), 8, m, f) == (size_t)m;
    std::fclose(f);
    if (!ok) { std::printf("short file %s\n", path); return 2; }
    cv::Matx34f pose;
    for (int i = 0; i < 12; ++i) pose.val[i] = -7.0f;                            // must stay untouched when the pose is rejected
    const bool accepted = SfMStereoUtilities::findCameraPoseFrom2D3DMatch(intrinsics(k), match, pose);
    std::printf("accepted %d\npose", accepted ? 1 : 0);
    for (int i = 0; i < 12; ++i) std::printf(" %a", (double)pose.val[i]);
    std::printf("\n");
    return 0;
}

int main(int argc, char** argv) {
    if (argc > 1) return from_file(argv[1]);
    const double canned[12][3] = {{4, 12, 50}, {12, 11, 55}, {22, 1, 45}, {13, 3, 60}, {11, 16, 61}, {21, 12, 65}, {24, 11, 67},
                                  {29, 6, 41}, {27, 4, 44}, {22, 7, 58}, {20, 9, 51}, {15, 10, 40}};
    const double d = M_PI / 180.0;                              // R = Rz(5) Ry(5) Rx(5), t = (-10, 0, 30): the fixture's left camera
    const double c = std::cos(5 * d), s = std::sin(5 * d);
    const double R[9] = {c * c, -s * c + c * s * s, s * s + c * s * c, s * c, c * c + s * s * s, -c * s + s * s * c, -s, c * s, c * c};
    const double t[3] = {-10, 0, 30};
    const float k[9] = {700, 0, 320, 0, 700, 240, 0, 0, 1};
    Image2D3DMatch match;
    for (int i = 0; i < 12; ++i) {
        double p[3];
        for (int r = 0; r < 3; ++r) p[r] = R[3 * r] * canned[i][0] + R[3 * r + 1] * canned[i][1] + R[3 * r + 2] * canned[i][2] + t[r];
        match.points3D.push_back(cv::Point3f((float)canned[i][0], (float)canned[i][1], (float)canned[i][2]));
        match.points2D.push_back(cv::Point2f((float)(700 * p[0] / p[2] + 320), (float)(700 * p[1] / p[2] + 240)));
    }
    cv::Matx34f pose;
    EXPECT(SfMStereoUtilities::findCameraPoseFrom2D3DMatch(intrinsics(k), match, pose), "the pose is accepted");
    double dr = 0, dt = 0;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) dr = std::fmax(dr, std::fabs(pose(i, j) - R[3 * i + j]));
        dt = std::fmax(dt, std::fabs(pose(i, 3) - t[i]));
    }
    EXPECT(dr < 0.01, "rotation within 0.01");
    EXPECT(dt < 0.1, "translation within 0.1");
    Image2D3DMatch scrambled = match;                            // every 2D point paired with another point's 3D point
    for (int i = 0; i < 12; ++i) scrambled.points3D[i] = match.points3D[(i * 5 + 3) % 12];
    cv::Matx34f untouched;
    for (int i = 0; i < 12; ++i) untouched.val[i] = -7.0f;
    EXPECT(!SfMStereoUtilities::findCameraPoseFrom2D3DMatch(intrinsics(k), scrambled, untouched), "scrambled matches are rejected");
    bool same = true;
    for (int i = 0; i < 12; ++i) same = same && untouched.val[i] == -7.0f;
    EXPECT(same, "a rejected pose is not written");
    std::printf("rotation error %.3g, translation error %.3g\n", dr, dt);
    std::printf(failures ? "SHIM_POSE_TEST FAIL (%d)\n" : "SHIM_POSE_TEST PASS\n", failures);
    return failures ? 1 : 0;
}
