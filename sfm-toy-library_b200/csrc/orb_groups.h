// orb_groups.h -- the per-image pyramid layout of ORB extraction (orb.cu) and how a batch of images is cut into groups that share one
// launch sequence.  Plain C++ with no CUDA types, so that tests/host_orb_groups.cpp can drive the same code with g++.
//
// Every image of a group has its own OrbLayout: its level sizes and its byte offsets into the group's arenas (pyramid, blurred
// pyramid and FAST scores share one offset; survivor masks, row counters and candidates have theirs).  A group is a run of
// consecutive images whose device bytes fit the device budget, whose pinned staging fits the staging budget and whose count fits grid z
// of the per-image launches.  An image over a budget on its own still gets a group of its own.  For equally sized images this is
// exactly `max(1, min(n, dev_budget / per_image, stage_budget / staging))` images per group, the rule of the equal-size batch.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <vector>

constexpr int ORB_LEVELS = 8;
constexpr int ORB_CHUNK = 32;                                  // pixels per survivor-mask word
constexpr size_t ORB_DEV_BUDGET = (size_t)2 << 30;             // device scratch of one group
constexpr size_t ORB_STAGE_BUDGET = (size_t)96 << 20;          // pinned staging of one group's host images
constexpr int ORB_MAX_GROUP = 65535;                           // grid z of the per-image launches

struct OrbLevel { int w, h, off, row0; float scale, inv_scale; int quota, taps; };   // taps: first resize tap of the level in the group's table
struct OrbLayout {
    OrbLevel lv[ORB_LEVELS];
    int total_rows;      // rows of all levels
    int slab;            // bytes of one image's pyramid (levels back to back, each 16-byte aligned)
    int chunks;          // survivor-mask words per row = ceil(level-0 width / 32), the same stride for every level
    int ncnt;            // total_rows * chunks
    int cand_cap;        // candidates the image can hold (3x3 suppression keeps at most one pixel of every 2x2 block)
    int src_stride;      // bytes per row of the B,G,R source
    const uint8_t* src;  // the B,G,R source on the device; null when grey input goes straight into level 0
    // where the image lives in its group's arenas
    size_t pix0;         // bytes before it in the pyramid, blurred pyramid and score arenas
    size_t mask0;        // survivor-mask words before it
    size_t cnt0;         // row counters (total_rows + 1 per image) before it
    size_t cand0;        // candidate records before it
};

// ORB_Impl::detectAndCompute: layerScale[l] = (float)pow((double)1.2f, l); layer size = cvRound(cols / scale) x cvRound(rows / scale);
// computeKeyPoints: nfeaturesPerLevel from the geometric series with factor 1 / 1.2f.  Offsets are left at zero.
inline void make_layout(int w, int h, int nfeatures, OrbLayout& L) {
    L = OrbLayout{};
    const double sf = (double)1.2f;
    int off = 0, row = 0;
    const float factor = (float)(1.0 / sf);
    float ndesired = (float)nfeatures * (1.0f - factor) / (1.0f - (float)std::pow((double)factor, (double)ORB_LEVELS));
    int sum = 0;
    for (int l = 0; l < ORB_LEVELS; l++) {
        OrbLevel& v = L.lv[l];
        v.scale = (float)std::pow(sf, (double)l);
        v.inv_scale = 1.0f / v.scale;
        v.w = (int)std::nearbyintf((float)w / v.scale); v.h = (int)std::nearbyintf((float)h / v.scale);
        if (v.w < 0) v.w = 0;
        if (v.h < 0) v.h = 0;
        if (v.w == 0 || v.h == 0) v.w = v.h = 0;
        v.off = off; v.row0 = row; v.taps = 0;
        off += (v.w * v.h + 15) & ~15; row += v.h;
        if (l < ORB_LEVELS - 1) { v.quota = (int)std::nearbyintf(ndesired); sum += v.quota; ndesired *= factor; }
        else v.quota = std::max(nfeatures - sum, 0);
    }
    L.total_rows = row; L.slab = (off + 255) & ~255; L.chunks = (w + ORB_CHUNK - 1) / ORB_CHUNK; L.ncnt = L.total_rows * L.chunks;
    L.cand_cap = L.slab / 4 + 64;
}

inline size_t orb_pad(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// Device bytes of one image: its B,G,R upload (raw_bytes, 0 when the image is already on the device or grey), pyramid, blurred pyramid,
// scores, survivor masks, row counters and offsets, level starts and candidates.
inline size_t orb_image_bytes(const OrbLayout& L, size_t raw_bytes) {
    return orb_pad(raw_bytes) + 3 * orb_pad((size_t)L.slab) + orb_pad(4 * (size_t)L.ncnt) + 2 * orb_pad(4 * (size_t)(L.total_rows + 1)) + orb_pad(64) +
           orb_pad(8 * (size_t)L.cand_cap);
}

// First image of every group, then n.  stage_bytes may be null (no staging).
inline std::vector<int> orb_groups(const size_t* dev_bytes, const size_t* stage_bytes, int n, size_t dev_budget = ORB_DEV_BUDGET,
                                   size_t stage_budget = ORB_STAGE_BUDGET, int max_images = ORB_MAX_GROUP) {
    std::vector<int> start{0};
    size_t dev = 0, stage = 0;
    int count = 0;
    for (int i = 0; i < n; ++i) {
        const size_t d = dev_bytes[i], s = stage_bytes ? stage_bytes[i] : 0;
        if (count && (dev + d > dev_budget || stage + s > stage_budget || count >= max_images)) { start.push_back(i); dev = stage = 0; count = 0; }
        dev += d; stage += s; ++count;
    }
    if (n > 0) start.push_back(n);
    return start;
}
