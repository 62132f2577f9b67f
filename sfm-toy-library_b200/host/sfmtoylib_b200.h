// sfmtoylib_b200.h -- declarations of the reference's stage boundary for a STANDALONE build of the shim (no reference
// tree, no OpenCV).  When the shim is built inside the reference tree (-DSFMB200_WITH_REFERENCE_HEADERS) the reference's
// own headers are used instead and this file is not included.
//
// Mirrors, name for name and argument for argument:
//   data carriers                         reference SfMToyLib/SfMCommon.h:55-99
//   SfM2DFeatureUtilities::extractFeatures reference SfMToyLib/SfM2DFeatureUtilities.h:38-42 (constructor, destructor, member function)
//   SfM2DFeatureUtilities::matchFeatures  reference SfMToyLib/SfM2DFeatureUtilities.h:44-46
//   SfMStereoUtilities::triangulateViews  reference SfMToyLib/SfMStereoUtilities.h:82-91
//   SfMBundleAdjustmentUtils::adjustBundle reference SfMToyLib/SfMBundleAdjustmentUtils.h:44-49
#pragma once
#ifdef SFMB200_WITH_OPENCV
#include <opencv2/core.hpp>
#include <opencv2/features2d.hpp>
#else
#include "cv_min.h"
#endif
#include <map>
#include <vector>

namespace sfmtoylib {

struct Intrinsics { cv::Mat K, Kinv, distortion; };
struct ImagePair { size_t left, right; };
typedef std::vector<cv::KeyPoint> Keypoints;
typedef std::vector<cv::Point2f> Points2f;
struct Features { Keypoints keyPoints; Points2f points; cv::Mat descriptors; };
struct Point3DInMap { cv::Point3f p; std::map<int, int> originatingViews; };
typedef std::vector<cv::DMatch> Matching;
typedef std::vector<Point3DInMap> PointCloud;
typedef cv::Matx34f Pose;

class SfM2DFeatureUtilities {
public:
    SfM2DFeatureUtilities();
    virtual ~SfM2DFeatureUtilities();
    Features extractFeatures(const cv::Mat& image);
    static Matching matchFeatures(const Features& featuresLeft, const Features& featuresRight);
};

struct Image2D3DMatch;        // sfm_glue.h (SfMCommon.h:71-74)

class SfMStereoUtilities {
public:
    static int findHomographyInliers(const Features& left, const Features& right, const Matching& matches);
    static bool findCameraMatricesFromMatch(const Intrinsics& intrinsics, const Matching& featureMatching, const Features& featuresLeft,
                                            const Features& featuresRight, Matching& prunedMatches, cv::Matx34f& Pleft, cv::Matx34f& Pright);
    static bool triangulateViews(const Intrinsics& intrinsics, const ImagePair imagePair, const Matching& matches,
                                 const Features& featuresLeft, const Features& featuresRight, const cv::Matx34f& Pleft,
                                 const cv::Matx34f& Pright, PointCloud& pointCloud);
    static bool findCameraPoseFrom2D3DMatch(const Intrinsics& intrinsics, const Image2D3DMatch& match, cv::Matx34f& cameraPose);
};

class SfMBundleAdjustmentUtils {
public:
    static void adjustBundle(PointCloud& pointCloud, std::vector<Pose>& cameraPoses, Intrinsics& intrinsics,
                             const std::vector<Features>& image2dFeatures);
};

}  // namespace sfmtoylib
