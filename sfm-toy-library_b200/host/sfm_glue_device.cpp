// sfm_glue_device.cpp -- DeviceGlue (sfm_glue.h): find2D3DMatches and mergeNewPointCloud over the C ABI's device glue.
#include "sfm_glue.h"
#include "../../include/sfmb200.h"
#include <stdexcept>
#include <string>

namespace sfmtoylib {

namespace {

void check(sfmb200_ctx* ctx, int rc, const char* what) {
    if (rc != SFMB200_OK) throw std::runtime_error(std::string(what) + ": " + sfmb200_last_error(ctx));
}

// a cloud as the C ABI takes it: coordinates, then the (view, feature) pairs of every point in ascending view order
struct FlatCloud {
    std::vector<float> X;
    std::vector<int32_t> off{0}, img, feat;
    explicit FlatCloud(const PointCloud& c) {
        X.reserve(3 * c.size()); off.reserve(c.size() + 1);
        for (const Point3DInMap& p : c) {
            X.push_back(p.p.x); X.push_back(p.p.y); X.push_back(p.p.z);
            for (const auto& kv : p.originatingViews) { img.push_back(kv.first); feat.push_back(kv.second); }
            off.push_back((int32_t)img.size());
        }
    }
};

}  // namespace

DeviceGlue::DeviceGlue(sfmb200_ctx* ctx, const std::vector<Features>& imageFeatures, const MatchMatrix& M)
    : ctx_(ctx), numImages_((int)imageFeatures.size()) {
    std::vector<int32_t> img_off{0}, pairs, q, t;
    std::vector<float> d;
    std::vector<int64_t> off{0};
    for (const Features& f : imageFeatures) img_off.push_back(img_off.back() + (int32_t)f.points.size());
    for (int i = 0; i < (int)M.size() && i < numImages_; ++i)
        for (int j = i + 1; j < (int)M[i].size() && j < numImages_; ++j) {
            if (M[i][j].empty()) continue;
            pairs.push_back(i); pairs.push_back(j);
            for (const cv::DMatch& m : M[i][j]) { q.push_back(m.queryIdx); t.push_back(m.trainIdx); d.push_back(m.distance); }
            off.push_back((int64_t)q.size());
        }
    check(ctx_, sfmb200_match_index_create(ctx_, img_off.data(), numImages_, pairs.data(), (int)pairs.size() / 2, q.data(), t.data(), d.data(),
                                           off.data(), &index_), "sfmb200_match_index_create");
}

DeviceGlue::~DeviceGlue() { sfmb200_match_index_destroy(index_); }

void DeviceGlue::setPair(int left, int right, const Matching& matches) {
    std::vector<int32_t> q, t;
    std::vector<float> d;
    for (const cv::DMatch& m : matches) { q.push_back(m.queryIdx); t.push_back(m.trainIdx); d.push_back(m.distance); }
    check(ctx_, sfmb200_match_index_set_pair(index_, left, right, q.data(), t.data(), d.data(), (int64_t)q.size()), "sfmb200_match_index_set_pair");
}

Images2D3DMatches DeviceGlue::find2D3DMatches(size_t numImages, const std::set<int>& doneViews, const std::vector<Features>& imageFeatures,
                                              const PointCloud& cloud) {
    if ((int)numImages != numImages_) throw std::runtime_error("find2D3DMatches: numImages differs from the index's image count");
    const FlatCloud fc(cloud);
    std::vector<uint8_t> done(numImages, 0);
    for (int v : doneViews) if (v >= 0 && (size_t)v < numImages) done[v] = 1;
    std::vector<int64_t> off(numImages + 1);
    for (int attempt = 0;; ++attempt) {
        const int rc = sfmb200_find_2d3d_matches(index_, done.data(), (int)cloud.size(), fc.off.data(), fc.img.data(), fc.feat.data(),
                                                 (int64_t)hitPoint_.size(), hitPoint_.data(), hitFeat_.data(), off.data());
        if (rc == SFMB200_ERR_INVALID && attempt == 0 && off[numImages] > (int64_t)hitPoint_.size()) {   // first call or a larger cloud
            hitPoint_.resize((size_t)off[numImages] + off[numImages] / 4); hitFeat_.resize(hitPoint_.size());
            continue;
        }
        check(ctx_, rc, "sfmb200_find_2d3d_matches");
        break;
    }
    Images2D3DMatches matches;
    for (size_t v = 0; v < numImages; ++v) {
        if (done[v]) continue;                                                   // SfM.cpp:476
        Image2D3DMatch& m = matches[(int)v];
        for (int64_t k = off[v]; k < off[v + 1]; ++k) {
            m.points2D.push_back(imageFeatures[v].points[hitFeat_[k]]);
            m.points3D.push_back(cloud[hitPoint_[k]].p);
        }
    }
    return matches;
}

MergeCounts DeviceGlue::mergeNewPointCloud(const PointCloud& cloud, PointCloud& recon, const MatchMatrix& M, MatchMatrix* mergeMatchMatrix) {
    const FlatCloud fe(recon), fn(cloud);
    std::vector<int8_t> outcome(cloud.size());
    std::vector<int32_t> target(cloud.size());
    int64_t counts[3] = {0, 0, 0};
    for (int attempt = 0;; ++attempt) {
        const int rc = sfmb200_merge_point_cloud(index_, (int)recon.size(), fe.X.data(), fe.off.data(), fe.img.data(), fe.feat.data(), (int)cloud.size(),
                                                 fn.X.data(), fn.off.data(), fn.img.data(), fn.feat.data(), (int64_t)logTarget_.size(), outcome.data(),
                                                 target.data(), logTarget_.data(), logView_.data(), logFeat_.data(), logOther_.data(), logPos_.data(), counts);
        if (rc == SFMB200_ERR_INVALID && attempt == 0 && counts[2] > (int64_t)logTarget_.size()) {
            const size_t n = (size_t)counts[2] + counts[2] / 4;
            for (auto* v : {&logTarget_, &logView_, &logFeat_, &logOther_, &logPos_}) v->resize(n);
            continue;
        }
        check(ctx_, rc, "sfmb200_merge_point_cloud");
        break;
    }
    for (size_t i = 0; i < cloud.size(); ++i) if (outcome[i] == SFMB200_MERGE_APPENDED) recon.push_back(cloud[i]);   // SfM.cpp:593
    for (int64_t k = 0; k < counts[2]; ++k) {
        recon[logTarget_[k]].originatingViews[logView_[k]] = logFeat_[k];                                              // :579
        if (mergeMatchMatrix) {
            const int l = std::min(logView_[k], logOther_[k]), r = std::max(logView_[k], logOther_[k]);
            (*mergeMatchMatrix)[l][r].push_back(M[l][r][logPos_[k]]);                                                   // :571
        }
    }
    MergeCounts c;
    c.newPoints = (size_t)counts[0]; c.mergedPoints = (size_t)counts[1];
    return c;
}

}  // namespace sfmtoylib
