// test_glue_device.cpp -- DeviceGlue (the device glue over the C ABI) against host/sfm_glue.cpp: the scenes of test_glue.cpp
// (same generator and seeds), hand-built scenes for each ordering rule of mergeNewPointCloud, a list replaced with setPair, and the
// refusals of the C ABI.  Usage: test_glue_device [seed] [--bench]
//   --bench: host glue against device glue on two scene sizes, one JSON line each (device times include flattening, upload,
//   download and applying the results).
#include "sfm_glue.h"
#include "../../include/sfmb200.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>

using namespace sfmtoylib;

struct Scene {
    size_t numImages;
    std::vector<Features> feats;
    MatchMatrix M;
    PointCloud recon, fresh;
    std::set<int> done;
};

// test_glue.cpp's generator, unchanged, so that the seeds give the same scenes
static Scene makeScene(unsigned seed, int V, int F, int nRecon, int nFresh, bool uniqueSorted) {
    std::mt19937 rng(seed);
    auto ri = [&](int lo, int hi) { return (int)(rng() % (unsigned)(hi - lo + 1)) + lo; };
    auto rf = [&](float lo, float hi) { return lo + (hi - lo) * (float)(rng() / 4294967296.0); };
    Scene s; s.numImages = (size_t)V;
    s.feats.resize(V);
    for (int v = 0; v < V; ++v) for (int f = 0; f < F; ++f) s.feats[v].points.push_back(cv::Point2f(rf(0, 1024), rf(0, 768)));
    s.M.assign(V, std::vector<Matching>(V));
    for (int i = 0; i < V; ++i)
        for (int j = i + 1; j < V; ++j) {
            Matching& m = s.M[i][j];
            if (uniqueSorted) {
                for (int q = 0; q < F; ++q) if (rng() % 3 == 0) m.push_back(cv::DMatch(q, ri(0, F - 1), 0, (float)ri(0, 60)));
            } else {
                const int n = F / 2;
                for (int k = 0; k < n; ++k) m.push_back(cv::DMatch(ri(0, F / 4), ri(0, F / 4), 0, (float)ri(0, 40)));
            }
        }
    auto randomPoint = [&](cv::Point3f centre, float spread) {
        Point3DInMap p; p.p = cv::Point3f(centre.x + rf(-spread, spread), centre.y + rf(-spread, spread), centre.z + rf(-spread, spread));
        const int k = ri(2, 4);
        while ((int)p.originatingViews.size() < k) p.originatingViews[ri(0, V - 1)] = ri(0, uniqueSorted ? F - 1 : F / 4);
        return p;
    };
    for (int i = 0; i < nRecon; ++i) s.recon.push_back(randomPoint(cv::Point3f(rf(-1, 1), rf(-1, 1), rf(4, 6)), 0.0f));
    for (int i = 0; i < nFresh; ++i) {
        const int mode = ri(0, 3);
        Point3DInMap p;
        if (mode == 0 || s.recon.empty()) p = randomPoint(cv::Point3f(rf(-1, 1), rf(-1, 1), rf(4, 6)), 0.0f);
        else {
            const Point3DInMap& e = s.recon[ri(0, (int)s.recon.size() - 1)];
            p = randomPoint(e.p, mode == 1 ? 0.004f : 0.012f);
            if (mode != 3) {
                auto it = e.originatingViews.begin(); std::advance(it, ri(0, (int)e.originatingViews.size() - 1));
                int nv = ri(0, V - 1); if (nv == it->first) nv = (nv + 1) % V;
                const int l = std::min(nv, it->first), r = std::max(nv, it->first);
                if (!s.M[l][r].empty()) {
                    const cv::DMatch& d = s.M[l][r][ri(0, (int)s.M[l][r].size() - 1)];
                    p.originatingViews.clear();
                    p.originatingViews[nv] = (nv == l) ? d.queryIdx : d.trainIdx;
                    const_cast<Point3DInMap&>(e).originatingViews[it->first] = (it->first == l) ? d.queryIdx : d.trainIdx;
                    p.originatingViews[ri(0, V - 1)] = ri(0, uniqueSorted ? F - 1 : F / 4);
                }
            }
        }
        s.fresh.push_back(p);
    }
    for (int v = 0; v < V; ++v) if (rng() % 2) s.done.insert(v);
    return s;
}

static bool samePoint(const cv::Point3f& a, const cv::Point3f& b) { return std::memcmp(&a, &b, sizeof a) == 0; }
static bool sameCloud(const PointCloud& a, const PointCloud& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i) if (!samePoint(a[i].p, b[i].p) || a[i].originatingViews != b[i].originatingViews) return false;
    return true;
}
static bool sameMatches(const MatchMatrix& a, const MatchMatrix& b) {
    for (size_t i = 0; i < a.size(); ++i) for (size_t j = 0; j < a[i].size(); ++j) {
        if (a[i][j].size() != b[i][j].size()) return false;
        for (size_t k = 0; k < a[i][j].size(); ++k)
            if (a[i][j][k].queryIdx != b[i][j][k].queryIdx || a[i][j][k].trainIdx != b[i][j][k].trainIdx ||
                std::memcmp(&a[i][j][k].distance, &b[i][j][k].distance, 4)) return false;
    }
    return true;
}
static bool same2D3D(const Images2D3DMatches& a, const Images2D3DMatches& b, size_t* pairs) {
    if (a.size() != b.size()) return false;
    *pairs = 0;
    for (const auto& kv : a) {
        auto it = b.find(kv.first);
        if (it == b.end() || it->second.points2D.size() != kv.second.points2D.size() || it->second.points3D.size() != kv.second.points3D.size()) return false;
        if (!kv.second.points2D.empty() && std::memcmp(kv.second.points2D.data(), it->second.points2D.data(), 8 * kv.second.points2D.size())) return false;
        if (!kv.second.points3D.empty() && std::memcmp(kv.second.points3D.data(), it->second.points3D.data(), 12 * kv.second.points3D.size())) return false;
        *pairs += kv.second.points2D.size();
    }
    return true;
}

struct MergeResult { PointCloud cloud; MatchMatrix dbg; MergeCounts c; };

static MergeResult hostMerge(const Scene& s) {
    const MatchIndex index(s.M);
    MergeResult r{s.recon, MatchMatrix(s.numImages, std::vector<Matching>(s.numImages)), {}};
    r.c = mergeNewPointCloud(s.fresh, r.cloud, s.M, index, &r.dbg);
    return r;
}
static MergeResult deviceMerge(DeviceGlue& g, const Scene& s) {
    MergeResult r{s.recon, MatchMatrix(s.numImages, std::vector<Matching>(s.numImages)), {}};
    r.c = g.mergeNewPointCloud(s.fresh, r.cloud, s.M, &r.dbg);
    return r;
}

// the device glue of `g` against the host glue on scene s: 2D-3D lists bitwise, merged cloud, counters, debug match matrix; the device
// merge twice (same outputs)
static int compare(sfmb200_ctx* ctx, DeviceGlue& g, const Scene& s, const char* what, MergeResult* out = nullptr) {
    (void)ctx;
    const MatchIndex index(s.M);
    const Images2D3DMatches ref = find2D3DMatches(s.numImages, s.done, s.M, index, s.feats, s.recon);
    const Images2D3DMatches got = g.find2D3DMatches(s.numImages, s.done, s.feats, s.recon);
    size_t pairs = 0;
    if (!same2D3D(ref, got, &pairs)) { printf("FAIL %s: 2D-3D lists differ\n", what); return 1; }
    const MergeResult h = hostMerge(s), d = deviceMerge(g, s), d2 = deviceMerge(g, s);
    if (h.c.newPoints != d.c.newPoints || h.c.mergedPoints != d.c.mergedPoints) {
        printf("FAIL %s: merge counters %zu/%zu vs %zu/%zu\n", what, h.c.newPoints, h.c.mergedPoints, d.c.newPoints, d.c.mergedPoints); return 1;
    }
    if (!sameCloud(h.cloud, d.cloud)) { printf("FAIL %s: merged cloud differs\n", what); return 1; }
    if (!sameMatches(h.dbg, d.dbg)) { printf("FAIL %s: merge match matrix differs\n", what); return 1; }
    if (!sameCloud(d.cloud, d2.cloud) || !sameMatches(d.dbg, d2.dbg)) { printf("FAIL %s: a second device merge differs\n", what); return 1; }
    printf("ok %s: %zu 2D-3D pairs, merge new=%zu merged=%zu dropped=%zu\n", what, pairs, d.c.newPoints, d.c.mergedPoints,
           s.fresh.size() - d.c.newPoints - d.c.mergedPoints);
    if (out) *out = d;
    return 0;
}

static int checkScene(sfmb200_ctx* ctx, const Scene& s, const char* what, MergeResult* out = nullptr) {
    DeviceGlue g(ctx, s.feats, s.M);
    return compare(ctx, g, s, what, out);
}

// ---- hand-built scenes: V views of F key points, lists set by hand
static Scene blank(int V, int F) {
    Scene s; s.numImages = (size_t)V; s.feats.resize(V);
    for (int v = 0; v < V; ++v) for (int f = 0; f < F; ++f) s.feats[v].points.push_back(cv::Point2f((float)(10 * v + f), (float)f));
    s.M.assign(V, std::vector<Matching>(V));
    return s;
}
static Point3DInMap pt(float x, float y, float z, std::map<int, int> views) { Point3DInMap p; p.p = cv::Point3f(x, y, z); p.originatingViews = views; return p; }

static int handScenes(sfmb200_ctx* ctx) {
    int fails = 0;
    MergeResult r;
    {   // two new points merging into one existing point
        Scene s = blank(4, 10);
        s.M[0][1] = {cv::DMatch(1, 2, 0, 5.f)}; s.M[0][2] = {cv::DMatch(1, 3, 0, 5.f)};
        s.recon = {pt(0, 0, 5, {{0, 1}})};
        s.fresh = {pt(0.001f, 0, 5, {{1, 2}, {3, 4}}), pt(0, 0.002f, 5, {{2, 3}})};
        fails += checkScene(ctx, s, "two new points into one existing point", &r);
        if (r.c.mergedPoints != 2 || r.cloud.size() != 1 || r.cloud[0].originatingViews.size() != 3) { printf("FAIL: expected two merges\n"); ++fails; }
    }
    {   // an insertion the same loop visits later: new key 5 goes in after existing key 0 and before 7, and (5, 7) then confirms
        Scene s = blank(8, 10);
        s.M[0][5] = {cv::DMatch(1, 4, 0, 1.f)}; s.M[5][7] = {cv::DMatch(9, 9, 0, 3.f), cv::DMatch(4, 6, 0, 2.f)};
        s.recon = {pt(1, 1, 5, {{0, 1}, {7, 6}})};
        s.fresh = {pt(1, 1, 5.003f, {{5, 4}})};
        fails += checkScene(ctx, s, "insertion visited by the same loop", &r);
        if (r.cloud[0].originatingViews.size() != 3) { printf("FAIL: expected the inserted key\n"); ++fails; }
    }
    {   // an overwrite of an existing key: (0, 2) confirms the new point's feature 7 in view 2, which replaces the existing 3
        Scene s = blank(4, 10);
        s.M[0][2] = {cv::DMatch(1, 7, 0, 0.f)}; s.M[2][3] = {cv::DMatch(7, 5, 0, 19.9f), cv::DMatch(3, 5, 0, 1.f)};
        s.recon = {pt(2, 2, 5, {{0, 1}, {2, 3}, {3, 5}})};
        s.fresh = {pt(2, 2.001f, 5, {{2, 7}})};
        fails += checkScene(ctx, s, "overwrite of an existing key", &r);
        if (r.cloud[0].originatingViews.at(2) != 7) { printf("FAIL: expected the overwrite\n"); ++fails; }
    }
    {   // a chain: the first new point is appended, the second merges into it, the third is near both but confirms nothing
        Scene s = blank(4, 10);
        s.M[1][2] = {cv::DMatch(2, 3, 0, 4.f)};
        s.recon = {pt(-3, 0, 5, {{0, 0}})};
        s.fresh = {pt(3, 0, 5, {{1, 2}}), pt(3.004f, 0, 5, {{2, 3}}), pt(3.002f, 0, 5, {{3, 1}})};
        fails += checkScene(ctx, s, "chain through an appended point", &r);
        if (r.c.newPoints != 1 || r.c.mergedPoints != 1 || r.cloud[1].originatingViews.size() != 2) { printf("FAIL: expected the chain\n"); ++fails; }
    }
    {   // distances within one float ulp of 0.01f (exact float differences): below merges, equal and above are no candidates (appended)
        Scene s = blank(3, 10);
        s.M[0][1] = {cv::DMatch(1, 1, 0, 1.f)};
        const float r0 = 0.01f, below = std::nextafter(r0, 0.f), above = std::nextafter(r0, 1.f);
        s.recon = {pt(0, 0, 0, {{0, 1}}), pt(0, 10, 0, {{0, 1}}), pt(0, 0, 20, {{0, 1}})};
        s.fresh = {pt(below, 0, 0, {{1, 1}}), pt(r0, 10, 0, {{1, 1}}), pt(above, 0, 20, {{1, 1}})};
        fails += checkScene(ctx, s, "distances one ulp around 0.01f", &r);
        if (r.c.mergedPoints != 1 || r.c.newPoints != 2) { printf("FAIL: expected one merge and two appends\n"); ++fails; }
    }
    return fails;
}

// a pair's list replaced with setPair equals an index created from the updated matrix, and the host glue on it
static int setPairCheck(sfmb200_ctx* ctx) {
    Scene s = makeScene(123, 7, 200, 400, 300, true);
    DeviceGlue g(ctx, s.feats, s.M);
    g.find2D3DMatches(s.numImages, s.done, s.feats, s.recon);
    for (auto lr : {std::make_pair(0, 3), std::make_pair(2, 6), std::make_pair(1, 2)}) {   // pruned, emptied, grown
        Matching& m = s.M[lr.first][lr.second];
        Matching next;
        if (lr.first == 0) { for (size_t k = 0; k < m.size(); k += 2) next.push_back(m[k]); }
        else if (lr.first == 1) { next = m; for (int q = 0; q < 200; q += 7) next.push_back(cv::DMatch(q, (q * 13) % 200, 0, 3.f)); }
        m = next;
        g.setPair(lr.first, lr.second, m);
    }
    int fails = compare(ctx, g, s, "lists replaced with setPair");
    fails += checkScene(ctx, s, "fresh index of the updated matrix");
    return fails;
}

static int expectInvalid(sfmb200_ctx* ctx, int rc, const char* what) {
    if (rc != SFMB200_ERR_INVALID) { printf("FAIL refusal %s: returned %d\n", what, rc); return 1; }
    printf("ok refusal %s: %s\n", what, sfmb200_last_error(ctx));
    return 0;
}

static int refusals(sfmb200_ctx* ctx) {
    int fails = 0;
    const int32_t img_off[4] = {0, 5, 10, 15};
    const int32_t q[2] = {1, 2}, t[2] = {3, 4};
    const float d[2] = {1.f, 2.f};
    const int64_t off[3] = {0, 1, 2};
    sfmb200_match_index* ix = nullptr;
    const int32_t lower[4] = {1, 0, 0, 2}, twice[4] = {0, 1, 0, 1}, diag[4] = {1, 1, 0, 2}, outside[4] = {0, 3, 0, 2};
    fails += expectInvalid(ctx, sfmb200_match_index_create(ctx, img_off, 3, lower, 2, q, t, d, off, &ix), "pair with left > right");
    fails += expectInvalid(ctx, sfmb200_match_index_create(ctx, img_off, 3, twice, 2, q, t, d, off, &ix), "pair listed twice");
    fails += expectInvalid(ctx, sfmb200_match_index_create(ctx, img_off, 3, diag, 2, q, t, d, off, &ix), "pair on the diagonal");
    fails += expectInvalid(ctx, sfmb200_match_index_create(ctx, img_off, 3, outside, 2, q, t, d, off, &ix), "pair naming image 3 of 3");
    const int32_t big_q[2] = {5, 2};
    const int32_t good[4] = {0, 1, 0, 2};
    fails += expectInvalid(ctx, sfmb200_match_index_create(ctx, img_off, 3, good, 2, big_q, t, d, off, &ix), "match outside the key points");
    fails += expectInvalid(ctx, sfmb200_match_index_create(ctx, img_off, 3, good, 2, q, t, nullptr, off, &ix), "no distances");
    if (sfmb200_match_index_create(ctx, img_off, 3, good, 2, q, t, d, off, &ix) != SFMB200_OK) { printf("FAIL: valid index refused\n"); return fails + 1; }
    fails += expectInvalid(ctx, sfmb200_match_index_set_pair(ix, 2, 1, q, t, d, 2), "set_pair with left > right");
    fails += expectInvalid(ctx, sfmb200_match_index_set_pair(ix, 0, 3, q, t, d, 2), "set_pair outside the images");
    fails += expectInvalid(ctx, sfmb200_match_index_set_pair(ix, 0, 1, t, big_q, d, 2), "set_pair match outside the key points");
    const uint8_t done[3] = {0, 0, 0};
    const float X[6] = {0, 0, 0, 1, 1, 1};
    int32_t outp[8], outf[8]; int64_t ooff[4];
    int8_t oc[2]; int32_t tg[2], lt[64], lv[64], lf[64], lo[64], lp[64]; int64_t cnt[3];
    struct Bad { const char* what; int32_t off[3], img[3], feat[3]; };
    const Bad bads[] = {{"view outside [0, n_img)", {0, 1, 2}, {0, 3, 0}, {0, 0, 0}},
                        {"feature outside its view's key points", {0, 1, 2}, {0, 1, 0}, {0, 5, 0}},
                        {"views not ascending", {0, 2, 2}, {1, 0, 0}, {0, 0, 0}},
                        {"negative feature", {0, 1, 2}, {0, 0, 0}, {-1, 0, 0}},
                        {"offsets not starting at 0", {1, 1, 2}, {0, 1, 0}, {0, 0, 0}}};
    for (const Bad& b : bads) {
        char w[128];
        snprintf(w, sizeof w, "find_2d3d_matches: %s", b.what);
        fails += expectInvalid(ctx, sfmb200_find_2d3d_matches(ix, done, 2, b.off, b.img, b.feat, 8, outp, outf, ooff), w);
        snprintf(w, sizeof w, "merge_point_cloud (existing): %s", b.what);
        const int32_t ok_off[3] = {0, 1, 2}, ok_img[2] = {0, 1}, ok_feat[2] = {1, 3};
        fails += expectInvalid(ctx, sfmb200_merge_point_cloud(ix, 2, X, b.off, b.img, b.feat, 2, X, ok_off, ok_img, ok_feat, 64, oc, tg, lt, lv, lf, lo, lp, cnt), w);
        snprintf(w, sizeof w, "merge_point_cloud (new): %s", b.what);
        fails += expectInvalid(ctx, sfmb200_merge_point_cloud(ix, 2, X, ok_off, ok_img, ok_feat, 2, X, b.off, b.img, b.feat, 64, oc, tg, lt, lv, lf, lo, lp, cnt), w);
    }
    // capacities below what the call found: the needed sizes come back, nothing is truncated
    const int32_t c_off[3] = {0, 1, 2}, c_img[2] = {0, 0}, c_feat[2] = {1, 1};
    fails += expectInvalid(ctx, sfmb200_find_2d3d_matches(ix, done, 2, c_off, c_img, c_feat, 1, outp, outf, ooff), "find_2d3d_matches: out_cap too small");
    if (ooff[3] != 2) { printf("FAIL: out_off[n_img] = %lld, expected 2\n", (long long)ooff[3]); ++fails; }
    const float Xn[6] = {0, 0, 0.001f, 5, 5, 5};
    const int32_t n_off[3] = {0, 1, 2}, n_img[2] = {1, 1}, n_feat[2] = {3, 3};
    fails += expectInvalid(ctx, sfmb200_merge_point_cloud(ix, 2, X, c_off, c_img, c_feat, 2, Xn, n_off, n_img, n_feat, 0, oc, tg, lt, lv, lf, lo, lp, cnt),
                           "merge_point_cloud: log_cap too small");
    if (cnt[2] != 1) { printf("FAIL: counts[2] = %lld, expected 1\n", (long long)cnt[2]); ++fails; }
    // the context and the index still work
    if (sfmb200_find_2d3d_matches(ix, done, 2, c_off, c_img, c_feat, 8, outp, outf, ooff) != SFMB200_OK || ooff[3] != 2 || outp[0] != 0 || outf[0] != 3) {
        printf("FAIL: a valid find_2d3d_matches after the refusals\n"); ++fails;
    }
    if (sfmb200_merge_point_cloud(ix, 2, X, c_off, c_img, c_feat, 2, Xn, n_off, n_img, n_feat, 64, oc, tg, lt, lv, lf, lo, lp, cnt) != SFMB200_OK ||
        cnt[0] != 1 || cnt[1] != 1 || cnt[2] != 1 || oc[0] != SFMB200_MERGE_MERGED || tg[0] != 0 || tg[1] != 2 || lt[0] != 0 || lv[0] != 1 || lf[0] != 3 ||
        lo[0] != 0 || lp[0] != 0) {
        printf("FAIL: a valid merge_point_cloud after the refusals\n"); ++fails;
    }
    sfmb200_match_index_destroy(ix);
    return fails;
}

static int bench(sfmb200_ctx* ctx, const char* name, const Scene& s, int features) {
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const int reps = 5;
    std::vector<double> hIdx, hFind, hMerge, dIdx, dFind, dMerge;
    Images2D3DMatches hm, dm;
    PointCloud hc, dc;
    MergeCounts hcnt, dcnt;
    for (int r = 0; r < reps + 1; ++r) {                                        // repetition 0 warms up and is not counted
        auto t0 = clk::now(); const MatchIndex index(s.M); auto t1 = clk::now();
        hm = find2D3DMatches(s.numImages, s.done, s.M, index, s.feats, s.recon); auto t2 = clk::now();
        hc = s.recon; auto t3 = clk::now(); hcnt = mergeNewPointCloud(s.fresh, hc, s.M, index); auto t4 = clk::now();
        DeviceGlue g(ctx, s.feats, s.M); auto t5 = clk::now();
        dm = g.find2D3DMatches(s.numImages, s.done, s.feats, s.recon); auto t6 = clk::now();
        dc = s.recon; auto t7 = clk::now(); dcnt = g.mergeNewPointCloud(s.fresh, dc, s.M); auto t8 = clk::now();
        if (r == 0) continue;
        hIdx.push_back(ms(t0, t1)); hFind.push_back(ms(t1, t2)); hMerge.push_back(ms(t3, t4));
        dIdx.push_back(ms(t4, t5)); dFind.push_back(ms(t5, t6)); dMerge.push_back(ms(t7, t8));
    }
    auto med = [](std::vector<double> v) { std::sort(v.begin(), v.end()); return v[v.size() / 2]; };
    size_t pairs = 0;
    const bool same = same2D3D(hm, dm, &pairs) && sameCloud(hc, dc) && hcnt.newPoints == dcnt.newPoints && hcnt.mergedPoints == dcnt.mergedPoints;
    printf("{\"scene\": \"%s\", \"views\": %zu, \"features_per_view\": %d, \"cloud_points\": %zu, \"new_points\": %zu, \"pairs\": %zu, "
           "\"merged\": %zu, \"host_index_ms\": %.3f, \"host_find2D3DMatches_ms\": %.3f, \"host_mergeNewPointCloud_ms\": %.3f, "
           "\"device_index_ms\": %.3f, \"device_find2D3DMatches_ms\": %.3f, \"device_mergeNewPointCloud_ms\": %.3f, \"identical\": %s}\n",
           name, s.numImages, features, s.recon.size(), s.fresh.size(), pairs, dcnt.mergedPoints, med(hIdx), med(hFind), med(hMerge), med(dIdx),
           med(dFind), med(dMerge), same ? "true" : "false");
    return same ? 0 : 1;
}

int main(int argc, char** argv) {
    const unsigned seed = argc > 1 && argv[1][0] != '-' ? (unsigned)atoi(argv[1]) : 1u;
    bool do_bench = false;
    for (int i = 1; i < argc; ++i) if (!strcmp(argv[i], "--bench")) do_bench = true;
    sfmb200_ctx* ctx = nullptr;
    if (sfmb200_create(0, &ctx) != SFMB200_OK) { printf("FAIL: sfmb200_create: %s\n", sfmb200_last_error(nullptr)); return 2; }
    int fails = 0;
    try {
        for (unsigned t = 0; t < 6; ++t) {
            char name[64];
            snprintf(name, sizeof name, "matcher-like scene %u", t);
            fails += checkScene(ctx, makeScene(seed * 100 + t, 5 + (int)t, 200, 400, 300, true), name);
            snprintf(name, sizeof name, "adversarial scene %u", t);
            fails += checkScene(ctx, makeScene(seed * 100 + 50 + t, 4 + (int)t, 60, 300, 300, false), name);
        }
        {
            Scene e; e.numImages = 3; e.feats.resize(3); e.M.assign(3, std::vector<Matching>(3));
            fails += checkScene(ctx, e, "empty scene");
        }
        fails += checkScene(ctx, makeScene(7, 24, 3000, 40000, 8000, true), "bench scene");
        fails += handScenes(ctx);
        fails += setPairCheck(ctx);
        fails += refusals(ctx);
        if (do_bench) {
            fails += bench(ctx, "test_glue --bench", makeScene(7, 24, 3000, 40000, 8000, true), 3000);
            fails += bench(ctx, "50 views", makeScene(11, 50, 5000, 200000, 20000, true), 5000);
        }
    } catch (const std::exception& e) {
        printf("FAIL: %s\n", e.what());
        ++fails;
    }
    sfmb200_destroy(ctx);
    printf(fails ? "FAILED (%d)\n" : "all device-glue checks passed\n", fails);
    return fails ? 1 : 0;
}
