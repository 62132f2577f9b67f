// match_cache.h -- bookkeeping and capacity plan of the per-call matcher's resident-image arena (sfmb200_match_knn2_ratio,
// match.cu).  Plain C++ with no CUDA types, so that tests/host_match_cache.cpp can drive the same code with g++.
//
// The arena is two growable device buffers: `desc` holds packed descriptor rows of ONE padded width, `exp` the expanded
// tensor-core operand blocks of 32-byte rows.  Images are bump-allocated at rows_used / blk_used and never moved; an arena
// that cannot take a call's new images is flushed whole.  Capacity rule, true after every plan:
//     rows_cap * width + 16 <= desc capacity (bytes),   blk_cap * block_bytes <= exp capacity (bytes)
// so an image placed while rows_used + rows <= rows_cap and blk_used + blocks <= blk_cap stays inside both buffers.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

struct MatchCacheEntry { const void* host; int rows; int desc_bytes; uint64_t hash; int row0; int blk0; };

struct MatchCacheState {
    int width = 0;                         // padded descriptor width (bytes) of the rows in the arena; 0 = capacities unknown
    int64_t rows_cap = 0, rows_used = 0;   // rows of `width` bytes the desc buffer holds / has handed out
    int blk_cap = 0, blk_used = 0;         // expanded blocks the exp buffer holds / has handed out
    std::vector<MatchCacheEntry> entries;
    int64_t hits = 0, misses = 0;

    // an image is resident when pointer, rows, width and content hash all match (a reused host buffer is a miss)
    const MatchCacheEntry* find(const void* host, int rows, int desc_bytes, uint64_t hash) const {
        for (const MatchCacheEntry& e : entries)
            if (e.host == host && e.rows == rows && e.desc_bytes == desc_bytes && e.hash == hash) return &e;
        return nullptr;
    }
    void flush() { entries.clear(); rows_used = 0; blk_used = 0; }
    // after a failed allocation the buffers' sizes are unknown here: the next plan starts from the buffers again
    void reset() { flush(); width = 0; rows_cap = 0; blk_cap = 0; }
};

constexpr int64_t MATCH_CACHE_MIN_ROWS = 16 * 8192;      // a grown arena has room for >= 16 images of 8 k features

// Byte sizes the two buffers must be reserved to before this call's images are placed (0: no growth needed).
struct MatchCachePlan { bool flushed; size_t desc_bytes, exp_bytes; };

// Plan one call matching q (nq rows) against t (nt rows), both desc_bytes wide and padded to `width` bytes, hashes hq / ht.
// desc_cap: the desc buffer's capacity in bytes now.  keep = false switches the arena off (every call starts empty).
// block_rows / block_bytes: rows per expanded block and its size (only 32-byte rows are expanded).
// Drops what cannot stay resident and sets rows_cap / blk_cap for the sizes returned; the caller reserves them.
inline MatchCachePlan match_cache_plan(MatchCacheState& s, size_t desc_cap, int width, bool keep, int desc_bytes, const void* q, int nq,
                                       uint64_t hq, const void* t, int nt, uint64_t ht, int block_rows, size_t block_bytes) {
    MatchCachePlan p = {false, 0, 0};
    if (width != s.width || !keep) {
        // rows of another width are of no use, and the rows the buffer holds depend on the width
        s.flush(); p.flushed = true;
        s.width = width;
        s.rows_cap = desc_cap >= 16 ? (int64_t)((desc_cap - 16) / width) : 0;
    }
    auto blocks = [&](int rows) { return width == 32 ? (rows + block_rows - 1) / block_rows : 0; };
    int64_t need_rows = 0; int need_blk = 0;
    if (!s.find(q, nq, desc_bytes, hq)) { need_rows += nq; need_blk += blocks(nq); }
    if (!s.find(t, nt, desc_bytes, ht) && !(t == q && nt == nq && ht == hq)) { need_rows += nt; need_blk += blocks(nt); }
    if (s.rows_used + need_rows > s.rows_cap || s.blk_used + need_blk > s.blk_cap) {
        // flush everything (simple and predictable), then grow if the arena cannot hold the pair or the minimum
        s.flush(); p.flushed = true;
        need_rows = (int64_t)nq + nt; need_blk = blocks(nq) + blocks(nt);
        const int64_t want_rows = std::max(need_rows, MATCH_CACHE_MIN_ROWS);
        if (s.rows_cap < want_rows) { p.desc_bytes = (size_t)want_rows * width + 16; s.rows_cap = want_rows; }
        const int want_blk = width == 32 ? std::max<int>(need_blk, (int)(want_rows / block_rows) + 32) : 0;
        if (want_blk > s.blk_cap) { p.exp_bytes = (size_t)want_blk * block_bytes; s.blk_cap = want_blk; }
    }
    return p;
}

// The host-side guard of every placement: the image's rows and blocks end inside the buffers.
inline bool match_cache_fits(const MatchCacheState& s, int rows, int nblk, int width, size_t block_bytes, size_t desc_cap, size_t exp_cap) {
    return (size_t)(s.rows_used + rows) * (size_t)width <= desc_cap && (size_t)(s.blk_used + nblk) * block_bytes <= exp_cap;
}
