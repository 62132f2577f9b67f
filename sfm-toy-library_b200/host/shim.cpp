// shim.cpp -- the stage functions of the reference, re-implemented as thin marshalling over the C ABI
// (include/sfmb200.h).  Linking this object instead of the bodies in the reference's
//   SfMToyLib/SfM2DFeatureUtilities.cpp:37-71 (constructor, extractFeatures, matchFeatures), SfMToyLib/SfMStereoUtilities.cpp:120-206,
//   SfMToyLib/SfMBundleAdjustmentUtils.cpp:99-222
// leaves SfM.cpp and main.cpp untouched (INTEGRATION.md).  No arithmetic happens here: only flattening of the
// std::vector / std::map / cv::Mat containers into the plain arrays of the ABI and back.
#ifdef SFMB200_WITH_REFERENCE_HEADERS
#include "SfMToyLib/SfM2DFeatureUtilities.h"
#include "SfMToyLib/SfMStereoUtilities.h"
#include "SfMToyLib/SfMBundleAdjustmentUtils.h"
#else
#include "sfmtoylib_b200.h"
#endif
#include "../../include/sfmb200.h"

#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <iostream>
#include <mutex>
#include <stdexcept>

namespace {

// One context per process (device from SFMB200_DEVICE, default 0), created on first use.  The library serialises
// concurrent calls internally, so the std::thread fan-out of SfM::createFeatureMatchMatrix (SfM.cpp:173-211) is safe.
sfmb200_ctx* context() {
    static sfmb200_ctx* ctx = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* dev = std::getenv("SFMB200_DEVICE");
        if (sfmb200_create(dev ? std::atoi(dev) : 0, &ctx) != SFMB200_OK) {
            std::cerr << "sfmb200: " << sfmb200_last_error(nullptr) << std::endl;
            throw std::runtime_error("sfmb200_create failed (no CPU fallback)");
        }
    });
    return ctx;
}

void check(int rc, const char* what) {
    if (rc != SFMB200_OK) {
        std::cerr << "sfmb200: " << what << ": " << sfmb200_last_error(context()) << std::endl;
        throw std::runtime_error(what);
    }
}

#if defined(SFMB200_WITH_REFERENCE_HEADERS) || defined(SFMB200_WITH_OPENCV)
const int kType8U = CV_8U;                    // OpenCV's macro
#else
const int kType8U = cv::CV_8U;                // cv_min.h
#endif
const double kNNMatchRatio = 0.8f;            // NN_MATCH_RATIO: the float literal widened to double
const float kMaxReprojectionError = 10.0f;    // MIN_REPROJECTION_ERROR

}  // namespace

namespace sfmtoylib {

#ifndef SFMB200_SHIM_KEEP_ORB     // define it to keep the reference's own constructor + extractFeatures (OpenCV's ORB) and replace only the matcher
// SfM2DFeatureUtilities.cpp:37-44: the reference creates the ORB detector and a matcher here; both live in libsfmb200.so now, the
// members (cv::Ptr, reference header :48-49) stay empty.
SfM2DFeatureUtilities::SfM2DFeatureUtilities() {}
SfM2DFeatureUtilities::~SfM2DFeatureUtilities() {}

// SfM2DFeatureUtilities.cpp:46-51: mDetector->detectAndCompute(image, noArray(), keyPoints, descriptors) with ORB::create(5000),
// then KeyPointsToPoints.  `image` is what cv::imread returned (8-bit B,G,R; SfM.cpp:124) or an 8-bit grey image.
Features SfM2DFeatureUtilities::extractFeatures(const cv::Mat& image) {
    static_assert(sizeof(cv::KeyPoint) == sizeof(sfmb200_keypoint), "cv::KeyPoint must be the 28-byte record of the ABI");
    Features features;
    if (image.empty()) return features;
    const cv::Mat img = image.isContinuous() ? image : image.clone();
    const int nfeatures = 5000;                                                    // ORB::create(5000), :39
    int cap = nfeatures + 64, n = 0;
    std::vector<sfmb200_keypoint> kp;
    std::vector<uint8_t> desc;
    for (;;) {
        kp.resize(cap); desc.resize(32 * (size_t)cap);
        check(sfmb200_orb_detect_and_compute(context(), img.ptr<uint8_t>(0), img.cols, img.rows, img.channels(), 0, nfeatures, cap, kp.data(),
                                             desc.data(), &n), "sfmb200_orb_detect_and_compute");
        if (n <= cap) break;
        cap = n;                                                                   // ties at a selection threshold: OpenCV returns them all
    }
    features.keyPoints.resize(n);
    if (n) std::memcpy((void*)features.keyPoints.data(), kp.data(), sizeof(sfmb200_keypoint) * (size_t)n);
    features.descriptors = cv::Mat(n, 32, kType8U);
    if (n) std::memcpy(features.descriptors.ptr<uint8_t>(0), desc.data(), 32 * (size_t)n);
    features.points.clear();                                                       // KeyPointsToPoints, SfMCommon.cpp:89-94
    for (const auto& k : features.keyPoints) features.points.push_back(k.pt);
    return features;
}
#endif  // SFMB200_SHIM_KEEP_ORB

Matching SfM2DFeatureUtilities::matchFeatures(const Features& featuresLeft, const Features& featuresRight) {
    // the ABI wants packed rows; a cv::Mat view (ROI, step > cols) is cloned first -- the reference accepts any cv::Mat
    const cv::Mat L = featuresLeft.descriptors.isContinuous() ? featuresLeft.descriptors : featuresLeft.descriptors.clone();
    const cv::Mat R = featuresRight.descriptors.isContinuous() ? featuresRight.descriptors : featuresRight.descriptors.clone();
    Matching out;
    if (L.rows == 0 || R.rows < 2) return out;
    const int bytes = (int)(L.cols * L.elemSize());
    std::vector<int32_t> q(L.rows), t(L.rows);
    std::vector<float> d(L.rows);
    int n = 0;
    check(sfmb200_match_knn2_ratio(context(), L.ptr<uint8_t>(0), L.rows, R.ptr<uint8_t>(0), R.rows, bytes, kNNMatchRatio,
                                   q.data(), t.data(), d.data(), &n), "sfmb200_match_knn2_ratio");
    out.reserve(n);
    for (int i = 0; i < n; ++i) out.push_back(cv::DMatch(q[i], t[i], 0, d[i]));      // knnMatch sets imgIdx = 0
    return out;
}

bool SfMStereoUtilities::triangulateViews(const Intrinsics& intrinsics, const ImagePair imagePair, const Matching& matches,
                                          const Features& featuresLeft, const Features& featuresRight, const cv::Matx34f& Pleft,
                                          const cv::Matx34f& Pright, PointCloud& pointCloud) {
    const int m = (int)matches.size();
    if (m == 0) return true;
    float K[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) K[3 * r + c] = intrinsics.K.at<float>(r, c);
    std::vector<int32_t> mq(m), mt(m);
    for (int i = 0; i < m; ++i) { mq[i] = matches[i].queryIdx; mt[i] = matches[i].trainIdx; }
    std::vector<float> X(3 * (size_t)m);
    std::vector<uint8_t> keep(m);
    int nkeep = 0;
    static_assert(sizeof(cv::Point2f) == 2 * sizeof(float), "Point2f must be two packed floats");
    check(sfmb200_triangulate(context(), K, Pleft.val, Pright.val,
                              reinterpret_cast<const float*>(featuresLeft.points.data()), (int)featuresLeft.points.size(),
                              reinterpret_cast<const float*>(featuresRight.points.data()), (int)featuresRight.points.size(),
                              mq.data(), mt.data(), m, kMaxReprojectionError, X.data(), keep.data(), &nkeep), "sfmb200_triangulate");
    pointCloud.reserve(pointCloud.size() + nkeep);
    for (int i = 0; i < m; ++i) {
        if (!keep[i]) continue;
        Point3DInMap p;
        p.p = cv::Point3f(X[3 * i], X[3 * i + 1], X[3 * i + 2]);
        p.originatingViews[(int)imagePair.left] = mq[i];
        p.originatingViews[(int)imagePair.right] = mt[i];
        pointCloud.push_back(p);
    }
    return true;
}

#ifdef SFMB200_SHIM_ESSENTIAL      // define it to replace findCameraMatricesFromMatch (OpenCV's findEssentialMat + recoverPose) too
// SfMStereoUtilities.cpp:74-118: essential-matrix RANSAC and pose recovery in one device call (sfmb200_find_camera_matrices).
bool SfMStereoUtilities::findCameraMatricesFromMatch(const Intrinsics& intrinsics, const Matching& matches, const Features& featuresLeft,
                                                     const Features& featuresRight, Matching& prunedMatches, cv::Matx34f& Pleft,
                                                     cv::Matx34f& Pright) {
    if (intrinsics.K.empty()) {
        std::cerr << "Intrinsics matrix (K) must be initialized." << std::endl;
        return false;
    }
    const int m = (int)matches.size();
    float K[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) K[3 * r + c] = intrinsics.K.at<float>(r, c);
    std::vector<int32_t> mq(m), mt(m);
    for (int i = 0; i < m; ++i) { mq[i] = matches[i].queryIdx; mt[i] = matches[i].trainIdx; }
    double R[9], t[3];
    std::vector<uint8_t> pose_mask(m);
    sfmb200_essential_summary summary;
    check(sfmb200_find_camera_matrices(context(), K, reinterpret_cast<const float*>(featuresLeft.points.data()), (int)featuresLeft.points.size(),
                                       reinterpret_cast<const float*>(featuresRight.points.data()), (int)featuresRight.points.size(),
                                       mq.data(), mt.data(), m, nullptr, nullptr, R, t, nullptr, pose_mask.data(), &summary),
          "sfmb200_find_camera_matrices");
    if (!summary.found) {
        std::cerr << "findCameraMatricesFromMatch: no essential matrix with more than 4 inliers among " << m << " matches" << std::endl;
        return false;
    }
    Pleft = cv::Matx34f::eye();
    for (int r = 0; r < 3; ++r) {                                                      // :105-107
        for (int c = 0; c < 3; ++c) Pright(r, c) = (float)R[3 * r + c];
        Pright(r, 3) = (float)t[r];
    }
    prunedMatches.clear();
    for (int i = 0; i < m; ++i)
        if (pose_mask[i]) prunedMatches.push_back(matches[i]);
    return true;
}
#endif  // SFMB200_SHIM_ESSENTIAL

#ifdef SFMB200_SHIM_HOMOGRAPHY     // define it to replace findHomographyInliers (OpenCV's findHomography(RANSAC)) too
// SfMStereoUtilities.cpp:51-72: cv::findHomography(RANSAC, RANSAC_THRESHOLD) -> countNonZero(mask), one device call
// (sfmb200_find_homography_pairs with one pair); the count is OpenCV's.  0 for fewer than 4 matches or no model.
int SfMStereoUtilities::findHomographyInliers(const Features& left, const Features& right, const Matching& matches) {
    const int m = (int)matches.size();
    if (m < 4) return 0;
    std::vector<float> pts(2 * (left.points.size() + right.points.size()));
    std::memcpy(pts.data(), left.points.data(), 2 * sizeof(float) * left.points.size());
    std::memcpy(pts.data() + 2 * left.points.size(), right.points.data(), 2 * sizeof(float) * right.points.size());
    const int32_t img_off[3] = {0, (int32_t)left.points.size(), (int32_t)(left.points.size() + right.points.size())};
    const int32_t pair[2] = {0, 1};
    const int64_t match_off[2] = {0, m};
    std::vector<int32_t> mq(m), mt(m);
    for (int i = 0; i < m; ++i) { mq[i] = matches[i].queryIdx; mt[i] = matches[i].trainIdx; }
    sfmb200_homography_options opt;
    sfmb200_homography_default_options(&opt);
    opt.threshold_px = 10.0;                                                            // RANSAC_THRESHOLD, SfMStereoUtilities.cpp:41
    sfmb200_homography_summary summary;
    check(sfmb200_find_homography_pairs(context(), pts.data(), img_off, 2, pair, 1, mq.data(), mt.data(), match_off, &opt, nullptr, nullptr, &summary),
          "sfmb200_find_homography_pairs");
    return summary.found ? summary.n_inliers : 0;
}
#endif  // SFMB200_SHIM_HOMOGRAPHY

void SfMBundleAdjustmentUtils::adjustBundle(PointCloud& pointCloud, std::vector<Pose>& cameraPoses, Intrinsics& intrinsics,
                                            const std::vector<Features>& image2dFeatures) {
    // dense numbering of the views that are actually observed (Ceres only knows blocks that appear in a residual)
    std::vector<int> dense(cameraPoses.size(), -1), used;
    for (const Point3DInMap& p : pointCloud)
        for (const auto& kv : p.originatingViews)
            if (dense[kv.first] < 0) dense[kv.first] = 0;
    for (size_t v = 0; v < cameraPoses.size(); ++v)
        if (dense[v] == 0) { dense[v] = (int)used.size(); used.push_back((int)v); }
    const int nc = (int)used.size(), np = (int)pointCloud.size();
    std::vector<double> cams(6 * (size_t)nc), pts(3 * (size_t)np);
    // reference :113-135: every non-empty pose becomes a 6-vector (float angle-axis of R, widened); an empty pose
    // (R diagonal exactly zero, :118-122) becomes CameraVector() = zeros and is never written back (:196-199)
    auto isEmpty = [](const Pose& pose) { return pose(0, 0) == 0 && pose(1, 1) == 0 && pose(2, 2) == 0; };
    auto toVector = [](const Pose& pose, double* v6) {
        float R[9], aa[3];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) R[3 * r + c] = pose(r, c);
        sfmb200_rotmat_to_angle_axis_f32(R, aa);                       // float conversion, then widened
        for (int k = 0; k < 3; ++k) { v6[k] = aa[k]; v6[3 + k] = pose(k, 3); }
    };
    for (int i = 0; i < nc; ++i) {
        const Pose& pose = cameraPoses[used[i]];
        if (isEmpty(pose)) continue;                                   // zeros, like CameraVector()
        toVector(pose, &cams[6 * i]);
    }
    double focal = intrinsics.K.at<float>(0, 0);
    const float cx = intrinsics.K.at<float>(0, 2), cy = intrinsics.K.at<float>(1, 2);
    std::vector<float> obs_xy;
    std::vector<int32_t> obs_cam, pt_off(np + 1, 0);
    for (int i = 0; i < np; ++i) {
        const Point3DInMap& p = pointCloud[i];
        pts[3 * i] = p.p.x; pts[3 * i + 1] = p.p.y; pts[3 * i + 2] = p.p.z;
        for (const auto& kv : p.originatingViews) {                    // std::map: ascending view id
            cv::Point2f p2d = image2dFeatures[kv.first].points[kv.second];
            p2d.x -= cx; p2d.y -= cy;                                  // float subtraction
            obs_xy.push_back(p2d.x); obs_xy.push_back(p2d.y);
            obs_cam.push_back(dense[kv.first]);
        }
        pt_off[i + 1] = (int32_t)obs_cam.size();
    }
    sfmb200_ba_options opt;
    sfmb200_ba_default_options(&opt);                                   // 500 iterations, 10 s, Ceres defaults
    opt.verbose = 1;                                                    // minimizer_progress_to_stdout = true
    sfmb200_ba_summary summary;
    check(sfmb200_ba_solve(context(), &opt, nc, np, (int)obs_cam.size(), cams.data(), pts.data(), &focal, obs_xy.data(),
                           obs_cam.data(), pt_off.data(), &summary), "sfmb200_ba_solve");
    std::cout << "sfmb200 BA: " << summary.message << " iterations " << summary.num_iterations << " cost "
              << summary.initial_cost << " -> " << summary.final_cost << "\n";
    if (summary.termination_type != SFMB200_BA_CONVERGENCE) {
        std::cerr << "Bundle adjustment failed." << std::endl;
        return;                                                         // inputs untouched
    }
    intrinsics.K.at<float>(0, 0) = (float)focal;
    intrinsics.K.at<float>(1, 1) = (float)focal;
    // reference :192-215: EVERY non-empty pose is rewritten from its 6-vector -- the observed ones from the optimised
    // parameters, the unobserved ones from their own (never optimised) float angle-axis, i.e. a round trip
    for (size_t v = 0; v < cameraPoses.size(); ++v) {
        Pose& pose = cameraPoses[v];
        if (isEmpty(pose)) continue;
        double v6[6], R[9];
        if (dense[v] >= 0) for (int k = 0; k < 6; ++k) v6[k] = cams[6 * (size_t)dense[v] + k];
        else toVector(pose, v6);
        sfmb200_angle_axis_to_rotmat(v6, R);
        for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) pose(r, c) = (float)R[3 * r + c]; pose(r, 3) = (float)v6[3 + r]; }
    }
    for (int i = 0; i < np; ++i) { pointCloud[i].p.x = (float)pts[3 * i]; pointCloud[i].p.y = (float)pts[3 * i + 1]; pointCloud[i].p.z = (float)pts[3 * i + 2]; }
}

}  // namespace sfmtoylib
