// host_orb_groups.cpp -- C entry points over sfm-toy-library_b200/csrc/orb_groups.h for tests/test_orb_groups_host.py (g++, no CUDA).
#include "../sfm-toy-library_b200/csrc/orb_groups.h"

extern "C" {

// device bytes of one w x h image with its B,G,R upload (raw = 1) or without it (raw = 0), and its pyramid rows
long long hog_image_bytes(int w, int h, int nfeatures, int raw, int* total_rows) {
    OrbLayout L;
    make_layout(w, h, nfeatures, L);
    if (total_rows) *total_rows = L.total_rows;
    return (long long)orb_image_bytes(L, raw ? (size_t)w * h * 3 : 0);
}

// groups of n images: writes the first image of every group and n into start[n + 1]; returns the number of groups
int hog_groups(const long long* dev_bytes, const long long* stage_bytes, int n, long long dev_budget, long long stage_budget, int max_images,
               int* start) {
    std::vector<size_t> d(dev_bytes, dev_bytes + n), s;
    if (stage_bytes) s.assign(stage_bytes, stage_bytes + n);
    const std::vector<int> g = orb_groups(d.data(), stage_bytes ? s.data() : nullptr, n, (size_t)dev_budget, (size_t)stage_budget, max_images);
    for (size_t i = 0; i < g.size(); ++i) start[i] = g[i];
    return (int)g.size() - 1;
}

long long hog_dev_budget() { return (long long)ORB_DEV_BUDGET; }
long long hog_stage_budget() { return (long long)ORB_STAGE_BUDGET; }
int hog_max_group() { return ORB_MAX_GROUP; }

}
