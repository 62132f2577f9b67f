// tests/host_match_cache.cpp -- TEST HARNESS: runs the per-call matcher's arena bookkeeping (csrc/match_cache.h) on the CPU the way
// sfmb200_match_knn2_ratio and cache_acquire (csrc/match.cu) do, without the copies: the two device buffers are modelled by their
// capacities under DevBuf::reserve's growth rule (csrc/common.cuh).  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/match_cache.h"

namespace {

constexpr int BLOCK_ROWS = 256;                // match_tc.cu: TC_N, rows per expanded block
constexpr size_t BLOCK_BYTES = 256 * 256;      // match_tc.cu: TcCfg<false>::BLOCK_BYTES, one block of 32-byte rows expanded to +-1 bytes

struct Arena : MatchCacheState { size_t desc_cap = 0, exp_cap = 0; };

void reserve(size_t& cap, size_t n) { if (n > cap) cap = n + n / 4 + 256; }      // DevBuf::reserve

int padded_width(int desc_bytes) {
    for (int w : {16, 32, 64, 128}) if (desc_bytes <= w) return w;
    return 0;
}

// cache_acquire without the copies: 0 = hit, 1 = miss placed, 2 = refused by the guard (the arena is reset, as match.cu does)
int acquire(Arena& a, const void* img, int rows, int desc_bytes, int width, uint64_t hash) {
    if (a.find(img, rows, desc_bytes, hash)) { a.hits++; return 0; }
    a.misses++;
    const int nblk = width == 32 ? (rows + BLOCK_ROWS - 1) / BLOCK_ROWS : 0;
    if (!match_cache_fits(a, rows, nblk, width, BLOCK_BYTES, a.desc_cap, a.exp_cap)) { a.reset(); return 2; }
    a.entries.push_back({img, rows, desc_bytes, hash, (int)a.rows_used, a.blk_used});
    a.rows_used += rows; a.blk_used += nblk;
    return 1;
}

}  // namespace

extern "C" {

int hmc_block_rows() { return BLOCK_ROWS; }
long long hmc_block_bytes() { return (long long)BLOCK_BYTES; }
void* hmc_new() { return new Arena(); }
void hmc_free(void* h) { delete static_cast<Arena*>(h); }

// One sfmb200_match_knn2_ratio call.  Returns 1 when the call returns before the arena (nq == 0 or nt < 2), else 0.
// out[14]: flushed, q (0 hit / 1 miss / 2 refused), t (same), width, rows_cap, rows_used, blk_cap, blk_used, desc capacity,
// exp capacity, hits, misses, desc bytes requested, exp bytes requested.
int hmc_call(void* h, const void* q, int nq, uint64_t hq, const void* t, int nt, uint64_t ht, int desc_bytes, int keep, long long* out) {
    Arena& a = *static_cast<Arena*>(h);
    for (int i = 0; i < 14; ++i) out[i] = -1;
    if (nq == 0 || nt < 2) return 1;
    const int width = padded_width(desc_bytes);
    const MatchCachePlan p = match_cache_plan(a, a.desc_cap, width, keep != 0, desc_bytes, q, nq, hq, t, nt, ht, BLOCK_ROWS, BLOCK_BYTES);
    reserve(a.desc_cap, p.desc_bytes);
    reserve(a.exp_cap, p.exp_bytes);
    out[0] = p.flushed;
    out[1] = acquire(a, q, nq, desc_bytes, width, hq);
    out[2] = out[1] == 2 ? 2 : acquire(a, t, nt, desc_bytes, width, ht);
    out[3] = a.width; out[4] = a.rows_cap; out[5] = a.rows_used; out[6] = a.blk_cap; out[7] = a.blk_used;
    out[8] = (long long)a.desc_cap; out[9] = (long long)a.exp_cap; out[10] = a.hits; out[11] = a.misses;
    out[12] = (long long)p.desc_bytes; out[13] = (long long)p.exp_bytes;
    return 0;
}

// Resident entries, 6 values each: host, rows, desc_bytes, hash, row0, blk0.  Returns how many there are (at most max are written).
int hmc_entries(void* h, long long* out, int max) {
    const Arena& a = *static_cast<Arena*>(h);
    int n = 0;
    for (const MatchCacheEntry& e : a.entries) {
        if (n < max) {
            long long* o = out + 6 * n;
            o[0] = (long long)(uintptr_t)e.host; o[1] = e.rows; o[2] = e.desc_bytes; o[3] = (long long)e.hash; o[4] = e.row0; o[5] = e.blk0;
        }
        ++n;
    }
    return n;
}

// Test hook: overstate the row capacity, as a planning mistake would, to exercise the guard.
void hmc_set_rows_cap(void* h, long long rows_cap) { static_cast<Arena*>(h)->rows_cap = rows_cap; }

}  // extern "C"
