// test_shim_essential_opencv.cpp -- C++ host-side test program of the shim built with SFMB200_SHIM_ESSENTIAL_OPENCV (runs on the
// GPU box): SfMStereoUtilities::findCameraMatricesFromMatch with cv::findEssentialMat's own samples, on image pairs read from a
// file; its Python test compares the pruned matches with cv2.findEssentialMat + cv2.recoverPose on the same pairs.
//   usage: test_shim_essential_opencv IN OUT
//   IN  (little-endian): int32 n_pairs, float K[9]; per pair: int32 n_left, float left[n_left][2], int32 n_right,
//       float right[n_right][2], int32 m, int32 queryIdx[m], int32 trainIdx[m]
//   OUT: per pair: int32 ok, int32 n_pruned, int32 queryIdx[n_pruned], int32 trainIdx[n_pruned], float Pright[12]
#include "sfmtoylib_b200.h"

#include <cstdio>
#include <vector>

using namespace sfmtoylib;

template <class T>
static bool get(std::FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }
template <class T>
static void put(std::FILE* f, const T* p, size_t n) { std::fwrite(p, sizeof(T), n, f); }

static bool readPoints(std::FILE* f, Features& feat) {
    int32_t n = 0;
    if (!get(f, &n, 1) || n < 0) return false;
    std::vector<float> xy(2 * (size_t)n);
    if (!get(f, xy.data(), xy.size())) return false;
    feat.points.clear();
    for (int32_t i = 0; i < n; ++i) feat.points.push_back(cv::Point2f(xy[2 * i], xy[2 * i + 1]));
    return true;
}

int main(int argc, char** argv) {
    if (argc != 3) { std::printf("usage: %s IN OUT\n", argv[0]); return 2; }
    std::FILE* in = std::fopen(argv[1], "rb");
    std::FILE* out = std::fopen(argv[2], "wb");
    if (!in || !out) { std::printf("cannot open the files\n"); return 2; }
    int32_t n_pairs = 0;
    float k[9];
    if (!get(in, &n_pairs, 1) || !get(in, k, 9)) { std::printf("bad input\n"); return 2; }
    Intrinsics intr; intr.K = cv::Mat(3, 3, cv::CV_32F);
    for (int i = 0; i < 9; ++i) intr.K.ptr<float>(0)[i] = k[i];
    int found = 0;
    for (int32_t p = 0; p < n_pairs; ++p) {
        Features left, right;
        int32_t m = 0;
        if (!readPoints(in, left) || !readPoints(in, right) || !get(in, &m, 1) || m < 0) { std::printf("bad input at pair %d\n", p); return 2; }
        std::vector<int32_t> q(m), t(m);
        if (!get(in, q.data(), m) || !get(in, t.data(), m)) { std::printf("bad input at pair %d\n", p); return 2; }
        Matching matching;
        for (int32_t i = 0; i < m; ++i) matching.push_back(cv::DMatch(q[i], t[i], 0));
        Matching pruned; cv::Matx34f Pl, Pr;
        const int32_t ok = SfMStereoUtilities::findCameraMatricesFromMatch(intr, matching, left, right, pruned, Pl, Pr) ? 1 : 0;
        found += ok;
        const int32_t n = (int32_t)pruned.size();
        std::vector<int32_t> pq(n), pt(n);
        for (int32_t i = 0; i < n; ++i) { pq[i] = pruned[i].queryIdx; pt[i] = pruned[i].trainIdx; }
        float P[12];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 4; ++c) P[4 * r + c] = ok ? Pr(r, c) : 0.0f;
        put(out, &ok, 1); put(out, &n, 1); put(out, pq.data(), n); put(out, pt.data(), n); put(out, P, 12);
    }
    std::fclose(in);
    if (std::fclose(out) != 0) { std::printf("cannot write the output\n"); return 2; }
    std::printf("SHIM_ESSENTIAL_OPENCV_TEST DONE %d pairs, %d with a pose\n", n_pairs, found);
    return 0;
}
