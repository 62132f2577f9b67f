// sfm_glue.h -- SURVEY.md 8(f-1): the two host-side scans of the reference's SfM driver that become the bottleneck once the
// three compute stages run on the GPU, with the same results and without the scans.
//
//   SfM::find2D3DMatches   (reference SfMToyLib/SfM.cpp:471-528): for every view not yet registered, every cloud point, every
//       originating (view, feature) of the point, a LINEAR scan of the pair's match list for the first match that touches the
//       feature.  O(views x points x k x matches-per-pair).
//   SfM::mergeNewPointCloud (reference SfMToyLib/SfM.cpp:530-600): for every new point a LINEAR scan of the whole cloud for
//       points closer than 0.01, then for every (new view, existing view) combination a linear scan of the pair's match list.
//       O(new x cloud + new x k^2 x matches-per-pair).
//
// Here the match lists are indexed once (MatchIndex: first occurrence per query index and per train index -- exactly what
// "first hit in list order, then break" (SfM.cpp:514, :519, :573) returns) and the cloud sits in a uniform grid of cell size
// >= the merge radius, searched in cloud order.  Every observable side effect of the reference loops is kept, including the
// insertion into existingPoint.originatingViews WHILE that map is being iterated (SfM.cpp:579) and the "near a cloud point
// but no confirming feature match => dropped" rule (SfM.cpp:591).  The reference's members become explicit arguments.
#pragma once
#include "sfmtoylib_b200.h"
#include <cstdint>
#include <map>
#include <set>
#include <unordered_map>
#include <vector>

struct sfmb200_ctx;
struct sfmb200_match_index;

namespace sfmtoylib {

typedef std::vector<std::vector<Matching>> MatchMatrix;                      // SfM.h:50 (upper triangular: [left][right], left < right)
struct Image2D3DMatch { Points2f points2D; std::vector<cv::Point3f> points3D; };   // SfMCommon.h:71-74
typedef std::map<int, Image2D3DMatch> Images2D3DMatches;                     // SfM.h:52

const float MERGE_CLOUD_POINT_MIN_MATCH_DISTANCE = 0.01f;                    // SfM.cpp:50
const float MERGE_CLOUD_FEATURE_MIN_MATCH_DISTANCE = 20.0f;                  // SfM.cpp:51

// Per pair: the positions of the matches grouped by query index (list order kept inside a group) and the first position of
// every train index.  matchFeatures emits every query index at most once, but nothing here relies on that.
class MatchIndex {
public:
    explicit MatchIndex(const MatchMatrix& m);
    // positions (ascending = list order) in matrix[left][right] of the matches with queryIdx == q: [*begin, *end)
    void byQuery(int left, int right, int q, const int32_t*& begin, const int32_t*& end) const {
        begin = end = nullptr;
        if (left < 0 || right < 0 || (size_t)left >= pairs_.size() || (size_t)right >= pairs_[left].size()) return;
        const Pair& p = pairs_[left][right];
        if (q < 0 || (size_t)q + 1 >= p.qoff.size()) return;
        begin = p.qpos.data() + p.qoff[q]; end = p.qpos.data() + p.qoff[q + 1];
    }
    // position of the first match with queryIdx == q (trainIdx == t), or -1
    int firstByQuery(int left, int right, int q) const { const int32_t *b, *e; byQuery(left, right, q, b, e); return b != e ? *b : -1; }
    int firstByTrain(int left, int right, int t) const {
        if (left < 0 || right < 0 || (size_t)left >= pairs_.size() || (size_t)right >= pairs_[left].size()) return -1;
        const Pair& p = pairs_[left][right];
        return (t >= 0 && (size_t)t < p.tfirst.size()) ? p.tfirst[t] : -1;
    }
private:
    struct Pair { std::vector<int32_t> qoff, qpos, tfirst; };                 // CSR by query index; first position per train index
    std::vector<std::vector<Pair>> pairs_;
};

// SfM::find2D3DMatches (SfM.cpp:471-528); numImages = mImages.size().
Images2D3DMatches find2D3DMatches(size_t numImages, const std::set<int>& doneViews, const MatchMatrix& featureMatchMatrix,
                                  const MatchIndex& index, const std::vector<Features>& imageFeatures, const PointCloud& reconstructionCloud);

struct MergeCounts { size_t newPoints = 0, mergedPoints = 0; };
// SfM::mergeNewPointCloud (SfM.cpp:530-600).  mergeMatchMatrix (the reference's debug visualisation input, :533, :571) is filled
// when non-null and already sized numImages x numImages.
MergeCounts mergeNewPointCloud(const PointCloud& cloud, PointCloud& reconstructionCloud, const MatchMatrix& featureMatchMatrix,
                               const MatchIndex& index, MatchMatrix* mergeMatchMatrix = nullptr);

// The same two functions on the GPU (host/sfm_glue_device.cpp over sfmb200_find_2d3d_matches / sfmb200_merge_point_cloud, linked
// with libsfmb200), with identical results.  The match index lives on the device: construct it after createFeatureMatchMatrix()
// and call setPair wherever the driver replaces a list (SfM.cpp:288, :431), since the index holds positions into the lists.
// Every call flattens the clouds once and applies the outcome; a failed call throws std::runtime_error with the library's message.
class DeviceGlue {
public:
    DeviceGlue(sfmb200_ctx* ctx, const std::vector<Features>& imageFeatures, const MatchMatrix& featureMatchMatrix);
    ~DeviceGlue();
    DeviceGlue(const DeviceGlue&) = delete;
    DeviceGlue& operator=(const DeviceGlue&) = delete;
    void setPair(int left, int right, const Matching& matches);
    Images2D3DMatches find2D3DMatches(size_t numImages, const std::set<int>& doneViews, const std::vector<Features>& imageFeatures,
                                      const PointCloud& reconstructionCloud);
    MergeCounts mergeNewPointCloud(const PointCloud& cloud, PointCloud& reconstructionCloud, const MatchMatrix& featureMatchMatrix,
                                   MatchMatrix* mergeMatchMatrix = nullptr);
private:
    sfmb200_ctx* ctx_;
    sfmb200_match_index* index_ = nullptr;
    int numImages_;
    std::vector<int32_t> hitPoint_, hitFeat_, logTarget_, logView_, logFeat_, logOther_, logPos_;   // reused, grown on demand
};

}  // namespace sfmtoylib
