// sfm_features.h -- the ABI's ORB records into the reference's Features container, shared by the stage shim's extractFeatures
// (shim.cpp) and sfmtoylib::readImagesAndFeatures (sfm_images.cpp).
#pragma once
#include "../../include/sfmb200.h"

#include <cstring>

namespace sfmtoylib {

// n key point records (the memory layout of cv::KeyPoint) and n 32-byte descriptors -> keyPoints, descriptors (CV_8U, n x 32) and
// points = KeyPointsToPoints(keyPoints) (SfMCommon.cpp:89-94).
inline Features featuresFromOrbRecords(const sfmb200_keypoint* kp, const uint8_t* desc, int n) {
    static_assert(sizeof(cv::KeyPoint) == sizeof(sfmb200_keypoint), "cv::KeyPoint must be the 28-byte record of the ABI");
#if defined(SFMB200_WITH_REFERENCE_HEADERS) || defined(SFMB200_WITH_OPENCV)
    const int type8U = CV_8U;                 // OpenCV's macro
#else
    const int type8U = cv::CV_8U;             // cv_min.h
#endif
    Features features;
    features.keyPoints.resize(n);
    if (n) std::memcpy((void*)features.keyPoints.data(), kp, sizeof(sfmb200_keypoint) * (size_t)n);
    features.descriptors = cv::Mat(n, 32, type8U);
    if (n) std::memcpy(features.descriptors.ptr<uint8_t>(0), desc, 32 * (size_t)n);
    features.points.clear();
    for (const auto& k : features.keyPoints) features.points.push_back(k.pt);
    return features;
}

}  // namespace sfmtoylib
