// glue.cu -- SURVEY.md 8(f-1) on the device: the match index, find2D3DMatches and mergeNewPointCloud of the reference driver
// (SfM.cpp:471-600) with host/sfm_glue.cpp's results.
//
// Match index.  One int32 pool holds, per pair (l, r) with l < r, the list and two lookup tables:
//     q[m] t[m] d[m] (float bits) | qpos[m]: positions grouped by query index, list order inside a group
//     qend[nf(l)]: group q is qpos[q ? qend[q-1] : 0 .. qend[q])  | tfirst[nf(r)]: first position of every train index, or -1
// One CTA builds one pair: counts and first positions with atomics (atomicMin is order-free), an exclusive scan, placement by
// atomic cursors, then every group of more than one position is sorted, so the result never depends on which thread came first.
// set_pair appends the new list to the pool and points the pair at it.
//
// find2D3DMatches.  One thread per (not-done view, cloud point) walks the point's views in ascending order and stops at the first
// hit; a scan over the hit flags gives every hit its place in (view, cloud) order, and the hits are written straight into pinned
// host memory, so the call downloads only what it found.
//
// mergeNewPointCloud.  Existing and new points go into a hashed uniform grid (cell 1.05 x 0.01f, CloudGrid's), each cell's points
// sorted by node id (existing points 0..ne-1 in cloud order, new point j as ne+j), so the points within cv::norm's radius of a new
// point come out of its 27 cells in the reference's candidate order.  New points that are neighbours, or share an existing
// neighbour, are joined by a union-find whose roots are the smallest node of each component: nothing one component does is seen by
// another.  One thread per component replays the reference's loop over its new points in order, keeping the maps' updates as an
// overlay log, while the components run side by side.  Scans then place the appended points and the log, which go straight into
// pinned host memory.
#include "common.cuh"
#include <algorithm>
#include <climits>

namespace {

struct PairRec { int64_t base; int32_t m, nq, nt; };    // m == 0: empty list (no tables)

constexpr int NT = 256;
constexpr int SC_PER = 8, SC_CH = NT * SC_PER;
constexpr uint64_t EMPTY_KEY = ~0ull;
constexpr float MERGE_FEATURE_DISTANCE = 20.0f;          // MERGE_CLOUD_FEATURE_MIN_MATCH_DISTANCE (SfM.cpp:51)
constexpr float MERGE_POINT_DISTANCE = 0.01f;            // MERGE_CLOUD_POINT_MIN_MATCH_DISTANCE (SfM.cpp:50)

// exclusive scan of one value per thread over a block of NT threads; *total = the block's sum
__device__ int32_t block_excl_scan(int32_t v, int32_t* sw, int32_t* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) sw[w] = x;
    __syncthreads();
    if (w == 0) {
        int32_t s = lane < NT / 32 ? sw[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
        if (lane < NT / 32) sw[lane] = s;
    }
    __syncthreads();
    const int32_t incl = x + (w ? sw[w - 1] : 0);
    *total = sw[NT / 32 - 1];
    __syncthreads();
    return incl - v;
}

// ---- device-wide exclusive scan of int32 counts (three launches: block sums, their scan, apply) ----
__global__ void __launch_bounds__(NT) scan_reduce_kernel(const int32_t* __restrict__ in, int n, int32_t* __restrict__ bsum) {
    __shared__ int32_t sw[NT / 32];
    const int64_t b = (int64_t)blockIdx.x * SC_CH + (int64_t)threadIdx.x * SC_PER;
    int32_t s = 0;
#pragma unroll
    for (int k = 0; k < SC_PER; ++k) if (b + k < n) s += in[b + k];
    int32_t tot;
    block_excl_scan(s, sw, &tot);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(NT) scan_sums_kernel(int32_t* __restrict__ bsum, int nb, int32_t* __restrict__ total) {
    __shared__ int32_t sw[NT / 32];
    int32_t carry = 0;
    for (int c = 0; c < nb; c += NT) {
        const int i = c + threadIdx.x;
        const int32_t v = i < nb ? bsum[i] : 0;
        int32_t tot;
        const int32_t ex = block_excl_scan(v, sw, &tot);
        if (i < nb) bsum[i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(NT) scan_apply_kernel(const int32_t* in, int n, const int32_t* __restrict__ bsum, int32_t* out) {
    __shared__ int32_t sw[NT / 32];
    const int64_t b = (int64_t)blockIdx.x * SC_CH + (int64_t)threadIdx.x * SC_PER;
    int32_t v[SC_PER], s = 0;
#pragma unroll
    for (int k = 0; k < SC_PER; ++k) { v[k] = b + k < n ? in[b + k] : 0; s += v[k]; }
    int32_t tot;
    int32_t run = block_excl_scan(s, sw, &tot) + bsum[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SC_PER; ++k) if (b + k < n) { out[b + k] = run; run += v[k]; }
}

// out[i] = sum of in[0..i) (in place allowed), *d_total = sum of all; bsum holds ceil(n / SC_CH) entries
int scan_excl(sfmb200_ctx* ctx, const int32_t* in, int n, int32_t* out, int32_t* bsum, int32_t* d_total) {
    if (n == 0) { SFM_CUDA(ctx, cudaMemsetAsync(d_total, 0, sizeof(int32_t), ctx->stream)); return SFMB200_OK; }
    const int nb = ceil_div(n, SC_CH);
    scan_reduce_kernel<<<nb, NT, 0, ctx->stream>>>(in, n, bsum);
    SFM_LAUNCH_CHECK(ctx);
    scan_sums_kernel<<<1, NT, 0, ctx->stream>>>(bsum, nb, d_total);
    SFM_LAUNCH_CHECK(ctx);
    scan_apply_kernel<<<nb, NT, 0, ctx->stream>>>(in, n, bsum, out);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

// ---- match index ----
__device__ __forceinline__ void sort_small(int32_t* a, int n) {           // insertion sort of one group / cell / list
    for (int i = 1; i < n; ++i) {
        const int32_t x = a[i];
        int j = i - 1;
        while (j >= 0 && a[j] > x) { a[j + 1] = a[j]; --j; }
        a[j + 1] = x;
    }
}

// one CTA per listed pair: copies the pair's list from src (q[m] t[m] d[m]) into the pool and builds qpos / qend / tfirst
__global__ void __launch_bounds__(NT) index_build_kernel(const PairRec* __restrict__ table, int32_t* __restrict__ pool,
                                                         const int32_t* __restrict__ build_pair, const int64_t* __restrict__ src_off,
                                                         const int32_t* __restrict__ src) {
    __shared__ int32_t sw[NT / 32];
    const PairRec P = table[build_pair[blockIdx.x]];
    const int m = P.m, nq = P.nq, nt = P.nt;
    int32_t* q = pool + P.base; int32_t* t = q + m; int32_t* d = t + m; int32_t* qpos = d + m; int32_t* qend = qpos + m;
    int32_t* tfirst = qend + nq;
    const int32_t* s = src + src_off[blockIdx.x];
    for (int k = threadIdx.x; k < m; k += NT) { q[k] = s[k]; t[k] = s[m + k]; d[k] = s[2 * m + k]; }
    for (int i = threadIdx.x; i < nq; i += NT) qend[i] = 0;
    for (int i = threadIdx.x; i < nt; i += NT) tfirst[i] = INT_MAX;
    __syncthreads();
    for (int k = threadIdx.x; k < m; k += NT) { atomicAdd(&qend[s[k]], 1); atomicMin(&tfirst[s[m + k]], k); }
    __syncthreads();
    int32_t carry = 0;
    for (int c = 0; c < nq; c += NT) {                                  // counts -> group starts
        const int i = c + threadIdx.x;
        const int32_t v = i < nq ? qend[i] : 0;
        int32_t tot;
        const int32_t ex = block_excl_scan(v, sw, &tot);
        if (i < nq) qend[i] = carry + ex;
        carry += tot;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < m; k += NT) qpos[atomicAdd(&qend[s[k]], 1)] = k;   // afterwards qend[q] = end of group q
    __syncthreads();
    for (int i = threadIdx.x; i < nq; i += NT) {
        const int lo = i ? qend[i - 1] : 0, hi = qend[i];
        if (hi - lo > 1) sort_small(qpos + lo, hi - lo);
    }
    for (int i = threadIdx.x; i < nt; i += NT) if (tfirst[i] == INT_MAX) tfirst[i] = -1;
}

// ---- find2D3DMatches ----
__global__ void __launch_bounds__(NT) find2d3d_kernel(const PairRec* __restrict__ table, const int32_t* __restrict__ pool, int n_img,
                                                      const int32_t* __restrict__ views, int np, const int32_t* __restrict__ voff,
                                                      const int32_t* __restrict__ vimg, const int32_t* __restrict__ vfeat,
                                                      int32_t* __restrict__ feat, int32_t* __restrict__ flag, int64_t ntask) {
    const int64_t g = (int64_t)blockIdx.x * NT + threadIdx.x;
    if (g >= ntask) return;
    const int v = views[g / np], i = (int)(g % np);
    int matched = -1;
    for (int k = voff[i]; k < voff[i + 1] && matched < 0; ++k) {
        const int ov = vimg[k], of = vfeat[k];
        if (ov < v) {                                                    // originating view on the left: first match of query `of`
            const PairRec P = table[(int64_t)ov * n_img + v];
            if (P.m) {
                const int32_t* qend = pool + P.base + 4 * (int64_t)P.m;
                const int lo = of ? qend[of - 1] : 0;
                if (qend[of] > lo) matched = pool[P.base + P.m + pool[P.base + 3 * (int64_t)P.m + lo]];
            }
        } else if (ov > v) {                                             // on the right: first match of train index `of`
            const PairRec P = table[(int64_t)v * n_img + ov];
            if (P.m) {
                const int pos = pool[P.base + 4 * (int64_t)P.m + P.nq + of];
                if (pos >= 0) matched = pool[P.base + pos];
            }
        }
    }
    feat[g] = matched;
    flag[g] = matched >= 0;
}

__global__ void __launch_bounds__(NT) find2d3d_write_kernel(const int32_t* __restrict__ feat, const int32_t* __restrict__ pos, int np,
                                                            int64_t ntask, int64_t cap, int32_t* out_point, int32_t* out_feat,
                                                            int32_t* vstart) {
    const int64_t g = (int64_t)blockIdx.x * NT + threadIdx.x;
    if (g >= ntask) return;
    if (g % np == 0) vstart[g / np] = pos[g];
    if (feat[g] >= 0 && pos[g] < cap) { out_point[pos[g]] = (int32_t)(g % np); out_feat[pos[g]] = feat[g]; }
}

// ---- mergeNewPointCloud ----
struct Cloud {                         // nodes 0..ne-1: existing points, ne..ne+nn-1: new points
    const float* P;                    // [(ne + nn) * 3]
    const int32_t *eoff, *eimg, *efeat, *noff, *nimg, *nfeat;
    int ne, nn;
    __device__ void map(int node, int& b, int& e, const int32_t*& img, const int32_t*& ft) const {
        if (node < ne) { b = eoff[node]; e = eoff[node + 1]; img = eimg; ft = efeat; }
        else { b = noff[node - ne]; e = noff[node - ne + 1]; img = nimg; ft = nfeat; }
    }
};

__device__ __forceinline__ long long cell_of(float v, double inv) { return (long long)floor(__dmul_rn((double)v, inv)); }
__device__ __forceinline__ uint64_t cell_key(long long a, long long b, long long c) {
    uint64_t h = (uint64_t)a * 0x9e3779b97f4a7c15ull ^ (uint64_t)b * 0xc2b2ae3d27d4eb4full ^ (uint64_t)c * 0x165667b19e3779f9ull;
    h ^= h >> 31; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 29;
    return h == EMPTY_KEY ? 0 : h;                                       // a shared key only adds candidates
}
// cv::norm(Point3f - Point3f) < 0.01f: float differences, squares, sum and root in double, no contraction
__device__ __forceinline__ bool within_radius(const float* a, const float* b) {
    const float dx = __fsub_rn(a[0], b[0]), dy = __fsub_rn(a[1], b[1]), dz = __fsub_rn(a[2], b[2]);
    const double s = __dadd_rn(__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)), __dmul_rn((double)dz, (double)dz));
    return __dsqrt_rn(s) < (double)MERGE_POINT_DISTANCE;
}
__device__ __forceinline__ uint32_t slot_hash(uint64_t k, uint32_t mask) { return (uint32_t)(k ^ (k >> 32)) & mask; }

__global__ void __launch_bounds__(NT) grid_insert_kernel(const float* __restrict__ P, int n, double inv, uint64_t* tkey, uint32_t mask,
                                                         int32_t* __restrict__ pslot, int32_t* cnt) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = cell_key(cell_of(P[3 * i], inv), cell_of(P[3 * i + 1], inv), cell_of(P[3 * i + 2], inv));
    uint32_t s = slot_hash(k, mask);
    for (;;) {
        const unsigned long long prev = atomicCAS((unsigned long long*)&tkey[s], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
        if (prev == EMPTY_KEY || prev == k) break;
        s = (s + 1) & mask;
    }
    pslot[i] = (int32_t)s;
    atomicAdd(&cnt[s], 1);
}

__global__ void __launch_bounds__(NT) grid_place_kernel(const int32_t* __restrict__ pslot, int n, int32_t* cursor, int32_t* __restrict__ cell_pts) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i < n) cell_pts[atomicAdd(&cursor[pslot[i]], 1)] = i;          // afterwards cursor[s] = end of cell s
}

// sorts every bucket [end[s] - cnt[s], end[s]) of items
__global__ void __launch_bounds__(NT) sort_buckets_kernel(const int32_t* __restrict__ end, const int32_t* __restrict__ cnt, int nb, int32_t* items) {
    const int s = blockIdx.x * NT + threadIdx.x;
    if (s < nb && cnt[s] > 1) sort_small(items + end[s] - cnt[s], cnt[s]);
}

// the grid slots of the (up to) 27 cells around a point; a slot two cells share through their key is listed once
struct Around { int32_t s[27]; int n; };
__device__ void cells_around(const float* p, double inv, const uint64_t* __restrict__ tkey, uint32_t mask, Around& A) {
    const long long x = cell_of(p[0], inv), y = cell_of(p[1], inv), z = cell_of(p[2], inv);
    A.n = 0;
    for (int a = -1; a <= 1; ++a)
        for (int b = -1; b <= 1; ++b)
            for (int c = -1; c <= 1; ++c) {
                const uint64_t k = cell_key((long long)((unsigned long long)x + a), (long long)((unsigned long long)y + b),
                                            (long long)((unsigned long long)z + c));
                uint32_t s = slot_hash(k, mask);
                while (tkey[s] != k && tkey[s] != EMPTY_KEY) s = (s + 1) & mask;
                if (tkey[s] == EMPTY_KEY) continue;
                bool dup = false;
                for (int u = 0; u < A.n; ++u) dup |= A.s[u] == (int32_t)s;
                if (!dup) A.s[A.n++] = (int32_t)s;
            }
}

struct Grid { const uint64_t* tkey; const int32_t *cend, *ccnt, *pts; uint32_t mask; double inv; };

// the smallest node above `after` within the radius of node `me` (itself excluded), or INT_MAX: the reference's candidates in
// cloud order, one at a time (each cell's points are sorted)
__device__ int next_neighbour(const Cloud& C, const Grid& G, const Around& A, int me, int after) {
    const float* p = C.P + 3 * (int64_t)me;
    int best = INT_MAX;
    for (int u = 0; u < A.n; ++u) {
        const int s = A.s[u];
        for (int j = G.cend[s] - G.ccnt[s]; j < G.cend[s]; ++j) {
            const int q = G.pts[j];
            if (q >= best) break;
            if (q <= after || q == me || !within_radius(C.P + 3 * (int64_t)q, p)) continue;
            best = q;
            break;
        }
    }
    return best;
}

__device__ int uf_find(int* parent, int x) {
    for (;;) {
        const int p = parent[x];
        if (p == x) return x;
        const int gp = parent[p];
        if (gp != p) atomicCAS(&parent[x], p, gp);
        x = p;
    }
}

__global__ void __launch_bounds__(NT) iota_kernel(int* a, int n) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i < n) a[i] = i;
}

// joins every new point with the nodes below it within the radius (the existing points it may merge into, the earlier new points
// it may merge into or share one with).  A root is only ever linked under a smaller root, so every component ends with its
// smallest node as root, whatever the order of the links.
__global__ void __launch_bounds__(NT) union_kernel(Cloud C, Grid G, int* parent) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i >= C.nn) return;
    const int me = C.ne + i;
    const float* p = C.P + 3 * (int64_t)me;
    Around A;
    cells_around(p, G.inv, G.tkey, G.mask, A);
    for (int u = 0; u < A.n; ++u)
        for (int j = G.cend[A.s[u]] - G.ccnt[A.s[u]]; j < G.cend[A.s[u]]; ++j) {
            const int q = G.pts[j];
            if (q >= me) break;
            if (!within_radius(C.P + 3 * (int64_t)q, p)) continue;
            int a = me, b = q;
            for (;;) {
                a = uf_find(parent, a); b = uf_find(parent, b);
                if (a == b) break;
                const int hi = a > b ? a : b, lo = a > b ? b : a;
                if (atomicCAS(&parent[hi], hi, lo) == hi) break;
            }
        }
}

__global__ void __launch_bounds__(NT) label_kernel(int ne, int nn, int* parent, int32_t* __restrict__ label, int32_t* gcnt) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i >= nn) return;
    label[i] = uf_find(parent, ne + i);
    atomicAdd(&gcnt[label[i]], 1);
}

__global__ void __launch_bounds__(NT) group_place_kernel(const int32_t* __restrict__ label, int nn, int32_t* cursor, int32_t* __restrict__ members) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i < nn) members[atomicAdd(&cursor[label[i]], 1)] = i;         // afterwards cursor[g] = end of component g
}

// the most log entries new point i can make: every one of its k views against every key of one map, which has at most n_img keys
__global__ void __launch_bounds__(NT) member_bound_kernel(const int32_t* __restrict__ members, int nn, const int32_t* __restrict__ noff, int n_img,
                                                          int32_t* __restrict__ bound) {
    const int at = blockIdx.x * NT + threadIdx.x;
    if (at < nn) bound[at] = (noff[members[at] + 1] - noff[members[at]]) * n_img;
}

struct Log { int32_t *target, *view, *feat, *other, *pos; };

// the first match of pair (l, r) with queryIdx == lf, trainIdx == rf and distance < 20 (SfM.cpp:566-575), or -1
__device__ int confirm(const PairRec* __restrict__ table, const int32_t* __restrict__ pool, int n_img, int l, int r, int lf, int rf) {
    if (l >= r) return -1;                                               // the diagonal is empty
    const PairRec P = table[(int64_t)l * n_img + r];
    if (!P.m) return -1;
    const int32_t* t = pool + P.base + P.m;
    const int32_t* d = t + P.m;
    const int32_t* qpos = d + P.m;
    const int32_t* qend = qpos + P.m;
    for (int j = lf ? qend[lf - 1] : 0; j < qend[lf]; ++j) {
        const int pos = qpos[j];
        if (t[pos] == rf && __int_as_float(d[pos]) < MERGE_FEATURE_DISTANCE) return pos;
    }
    return -1;
}

// the live map of `node`: its own entries, overwritten and extended by the log entries [lo, hi) of its component
__device__ int map_next_key(const Cloud& C, const Log& L, int lo, int hi, int node, int after) {
    int b, e; const int32_t *img, *ft;
    C.map(node, b, e, img, ft);
    int best = INT_MAX;
    for (int k = b; k < e; ++k) if (img[k] > after) { best = img[k]; break; }
    for (int k = lo; k < hi; ++k) if (L.target[k] == node && L.view[k] > after && L.view[k] < best) best = L.view[k];
    return best;
}
__device__ int map_value(const Cloud& C, const Log& L, int lo, int hi, int node, int key) {
    for (int k = hi - 1; k >= lo; --k) if (L.target[k] == node && L.view[k] == key) return L.feat[k];
    int b, e; const int32_t *img, *ft;
    C.map(node, b, e, img, ft);
    for (int k = b; k < e; ++k) if (img[k] == key) return ft[k];
    return -1;
}

// one thread per component: the reference's loop (SfM.cpp:541-598) over the component's new points in order.  Its log entries go to
// [bstart[first member], ...), which the bounds of its members reserve.
__global__ void __launch_bounds__(128) resolve_kernel(Cloud C, Grid G, const PairRec* __restrict__ table, const int32_t* __restrict__ pool, int n_img,
                                                      const int32_t* __restrict__ gend, const int32_t* __restrict__ gcnt,
                                                      const int32_t* __restrict__ members, const int32_t* __restrict__ bstart, uint8_t* appended,
                                                      int32_t* __restrict__ kind, int32_t* __restrict__ tnode, int32_t* __restrict__ lfirst,
                                                      int32_t* __restrict__ lcnt, Log L) {
    const int g = blockIdx.x * 128 + threadIdx.x;
    if (g >= C.ne + C.nn || gcnt[g] == 0) return;
    const int m0 = gend[g] - gcnt[g], m1 = gend[g];
    const int lo = bstart[m0];
    int head = lo;
    for (int mi = m0; mi < m1; ++mi) {
        const int i = members[mi], me = C.ne + i;
        Around A;
        cells_around(C.P + 3 * (int64_t)me, G.inv, G.tkey, G.mask, A);
        const int first = head;
        bool near = false, any = false;
        int target = -1;
        for (int c = next_neighbour(C, G, A, me, -1); c != INT_MAX && !any; c = next_neighbour(C, G, A, me, c)) {
            if (c >= C.ne && (c > me || !appended[c - C.ne])) continue;   // the grid holds the existing and the appended points
            near = true;
            for (int nk = C.noff[i]; nk < C.noff[i + 1]; ++nk) {
                const int a = C.nimg[nk], fa = C.nfeat[nk];
                // std::map iteration while the loop inserts into the same map (:579): the next key is the smallest one above the current
                for (int b = map_next_key(C, L, lo, head, c, -1); b != INT_MAX; b = map_next_key(C, L, lo, head, c, b)) {
                    const int fb = map_value(C, L, lo, head, c, b);
                    const int pos = a < b ? confirm(table, pool, n_img, a, b, fa, fb) : confirm(table, pool, n_img, b, a, fb, fa);
                    if (pos >= 0) {
                        L.target[head] = c; L.view[head] = a; L.feat[head] = fa; L.other[head] = b; L.pos[head] = pos;
                        ++head;
                        any = true;
                    }
                }
            }
            if (any) target = c;
        }
        if (any) { kind[i] = SFMB200_MERGE_MERGED; tnode[i] = target; }
        else if (!near) { kind[i] = SFMB200_MERGE_APPENDED; tnode[i] = me; appended[i] = 1; }
        else { kind[i] = SFMB200_MERGE_DROPPED; tnode[i] = -1; }
        lfirst[i] = first; lcnt[i] = head - first;
    }
}

__global__ void __launch_bounds__(NT) appended_flags_kernel(const uint8_t* __restrict__ appended, int nn, int32_t* __restrict__ f) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i < nn) f[i] = appended[i];
}

// outcome and log into pinned host memory: the cloud index of a node is the node itself (existing point) or ne + its rank among the
// appended points
__global__ void __launch_bounds__(NT) merge_write_kernel(int ne, int nn, const int32_t* __restrict__ kind, const int32_t* __restrict__ tnode,
                                                         const int32_t* __restrict__ apos, const int32_t* __restrict__ lfirst,
                                                         const int32_t* __restrict__ lcnt, const int32_t* __restrict__ loff, Log L, int64_t cap,
                                                         int8_t* out_kind, int32_t* out_target, Log O) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i >= nn) return;
    auto cloud_index = [&](int node) { return node < ne ? node : ne + apos[node - ne]; };
    out_kind[i] = (int8_t)kind[i];
    out_target[i] = tnode[i] < 0 ? -1 : cloud_index(tnode[i]);
    for (int s = 0; s < lcnt[i]; ++s) {
        const int64_t at = (int64_t)loff[i] + s, from = lfirst[i] + s;
        if (at >= cap) break;
        O.target[at] = cloud_index(L.target[from]); O.view[at] = L.view[from]; O.feat[at] = L.feat[from];
        if (O.other) O.other[at] = L.other[from];
        if (O.pos) O.pos[at] = L.pos[from];
    }
}

}  // namespace

struct sfmb200_match_index {
    sfmb200_ctx* ctx = nullptr;
    int n_img = 0;
    std::vector<int32_t> img_off;
    std::vector<PairRec> table;        // host mirror of d_table [n_img * n_img]
    DevBuf d_table;
    int32_t* pool = nullptr;           // device, int32 words
    int64_t pool_cap = 0, pool_used = 0;
    ~sfmb200_match_index() { d_table.release(); if (pool) cudaFree(pool); }
};

namespace {

int64_t pair_words(int64_t m, int nq, int nt) { return m ? 4 * m + nq + nt : 0; }

struct PairList { int l, r; const int32_t *q, *t; const float* d; int64_t m; };

// points the listed pairs at fresh space at the end of the pool (growing it), uploads their lists and builds their tables; one host
// synchronisation.  The space a replaced list held is not reused: set_pair is called for a few pairs per added view.
int index_load(sfmb200_match_index* ix, const std::vector<PairList>& lists) {
    sfmb200_ctx* ctx = ix->ctx;
    int64_t need = 0, M = 0;
    std::vector<int32_t> build;
    std::vector<int64_t> src_off;
    for (const PairList& L : lists) {
        PairRec& R = ix->table[(size_t)L.l * ix->n_img + L.r];
        R.m = (int32_t)L.m; R.nq = ix->img_off[L.l + 1] - ix->img_off[L.l]; R.nt = ix->img_off[L.r + 1] - ix->img_off[L.r];
        R.base = ix->pool_used + need;
        need += pair_words(L.m, R.nq, R.nt);
        if (L.m) { build.push_back(L.l * ix->n_img + L.r); src_off.push_back(3 * M); M += L.m; }
    }
    if (ix->pool_used + need > ix->pool_cap) {
        const int64_t cap = std::max<int64_t>(2 * (ix->pool_used + need), 1 << 16);
        int32_t* np = nullptr;
        SFM_CUDA(ctx, cudaMalloc(&np, 4 * (size_t)cap));
        if (ix->pool_used) SFM_CUDA(ctx, cudaMemcpyAsync(np, ix->pool, 4 * (size_t)ix->pool_used, cudaMemcpyDeviceToDevice, ctx->stream));
        SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ix->pool) cudaFree(ix->pool);
        ix->pool = np; ix->pool_cap = cap;
    }
    ix->pool_used += need;
    const size_t nt = ix->table.size(), nbld = build.size();
    const size_t bytes = Carver::pad(sizeof(PairRec) * nt) + Carver::pad(4 * nbld) + Carver::pad(8 * nbld) + Carver::pad(12 * (size_t)M) + 256;
    SFM_CUDA(ctx, ctx->pinned.reserve(bytes));
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    SFM_CUDA(ctx, ix->d_table.reserve(sizeof(PairRec) * nt));
    Carver hc(ctx->pinned.p), dc(ctx->scratch.p);
    PairRec* h_tab = hc.take<PairRec>(nt); int32_t* h_b = hc.take<int32_t>(nbld); int64_t* h_so = hc.take<int64_t>(nbld);
    int32_t* h_src = hc.take<int32_t>(3 * (size_t)M);
    const PairRec* d_tab = dc.take<PairRec>(nt); const int32_t* d_b = dc.take<int32_t>(nbld); const int64_t* d_so = dc.take<int64_t>(nbld);
    const int32_t* d_src = dc.take<int32_t>(3 * (size_t)M);
    memcpy(h_tab, ix->table.data(), sizeof(PairRec) * nt);
    if (nbld) { memcpy(h_b, build.data(), 4 * nbld); memcpy(h_so, src_off.data(), 8 * nbld); }
    int64_t at = 0;
    for (const PairList& L : lists) {
        if (!L.m) continue;
        memcpy(h_src + at, L.q, 4 * (size_t)L.m); memcpy(h_src + at + L.m, L.t, 4 * (size_t)L.m); memcpy(h_src + at + 2 * L.m, L.d, 4 * (size_t)L.m);
        at += 3 * L.m;
    }
    SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, ctx->pinned.p, hc.off, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(ix->d_table.p, d_tab, sizeof(PairRec) * nt, cudaMemcpyDeviceToDevice, ctx->stream));
    if (nbld) {
        index_build_kernel<<<(int)nbld, NT, 0, ctx->stream>>>((const PairRec*)ix->d_table.p, ix->pool, d_b, d_so, d_src);
        SFM_LAUNCH_CHECK(ctx);
    }
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SFMB200_OK;
}

// a cloud's view lists: offsets from 0, monotone; views strictly ascending in [0, n_img); features inside their image's key points
int check_views(sfmb200_ctx* ctx, const char* what, int n, const int32_t* off, const int32_t* img, const int32_t* feat,
                const std::vector<int32_t>& img_off) {
    const int n_img = (int)img_off.size() - 1;
    if (!off) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: null buffer", what);
    if (off[0] != 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: view offsets must start at 0", what);
    for (int i = 0; i < n; ++i) if (off[i + 1] < off[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: view offsets not monotone at point %d", what, i);
    if (off[n] > 0 && (!img || !feat)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: null buffer", what);
    for (int i = 0; i < n; ++i)
        for (int k = off[i]; k < off[i + 1]; ++k) {
            const int v = img[k];
            if (v < 0 || v >= n_img) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: point %d names view %d outside [0, %d)", what, i, v, n_img);
            if (k > off[i] && v <= img[k - 1]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: views of point %d are not strictly ascending", what, i);
            if (feat[k] < 0 || feat[k] >= img_off[v + 1] - img_off[v])
                return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%s: point %d names feature %d outside the key points of view %d", what, i, feat[k], v);
        }
    return SFMB200_OK;
}

int check_list(sfmb200_ctx* ctx, const sfmb200_match_index* ix, int l, int r, const int32_t* q, const int32_t* t, const float* d, int64_t m) {
    if (l < 0 || r < 0 || l >= ix->n_img || r >= ix->n_img) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair (%d, %d) names an image outside [0, %d)", l, r, ix->n_img);
    if (l >= r) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair (%d, %d): the match matrix is upper-triangular, left < right", l, r);
    if (m < 0 || m > INT32_MAX / 4) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair (%d, %d): %lld matches", l, r, (long long)m);
    if (m > 0 && (!q || !t || !d)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    const int nl = ix->img_off[l + 1] - ix->img_off[l], nr = ix->img_off[r + 1] - ix->img_off[r];
    for (int64_t k = 0; k < m; ++k)
        if (q[k] < 0 || q[k] >= nl || t[k] < 0 || t[k] >= nr)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match %lld of pair (%d, %d) indexes outside its images' key points", (long long)k, l, r);
    return SFMB200_OK;
}

}  // namespace

extern "C" {

int sfmb200_match_index_create(sfmb200_ctx* ctx, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs, const int32_t* match_q,
                               const int32_t* match_t, const float* match_d, const int64_t* match_off, sfmb200_match_index** index) {
    if (!ctx || !index) return SFMB200_ERR_INVALID;
    *index = nullptr;
    if (n_img < 0 || n_pairs < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "negative n_img or n_pairs");
    if (n_img > 1024) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%d images: at most 1024", n_img);
    int64_t M = 0;
    // the index reads no key point coordinates: img_off stands in for the pts array the batch check asks for
    if (const int rc = check_pair_batch(ctx, (const float*)img_off, img_off, n_img, pairs, n_pairs, match_q, match_t, match_off, INT32_MAX / 4, &M))
        return rc;
    if (M > 0 && !match_d) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    std::vector<uint8_t> seen((size_t)n_img * n_img, 0);
    for (int p = 0; p < n_pairs; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        if (l >= r) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair %d (%d, %d): the match matrix is upper-triangular, left < right", p, l, r);
        if (seen[(size_t)l * n_img + r]++) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair %d (%d, %d) appears twice", p, l, r);
    }
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    sfmb200_match_index* ix = new sfmb200_match_index();
    ix->ctx = ctx; ix->n_img = n_img;
    ix->img_off.assign(img_off, img_off + n_img + 1);
    ix->table.assign((size_t)n_img * n_img, PairRec{0, 0, 0, 0});
    std::vector<PairList> lists;
    for (int p = 0; p < n_pairs; ++p)
        lists.push_back({pairs[2 * p], pairs[2 * p + 1], match_q + match_off[p], match_t + match_off[p], match_d + match_off[p],
                         match_off[p + 1] - match_off[p]});
    const int rc = n_img ? index_load(ix, lists) : SFMB200_OK;
    if (rc) { delete ix; return rc; }
    *index = ix;
    return SFMB200_OK;
}

int sfmb200_match_index_set_pair(sfmb200_match_index* ix, int left, int right, const int32_t* match_q, const int32_t* match_t, const float* match_d,
                                 int64_t m) {
    if (!ix) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = ix->ctx;
    if (const int rc = check_list(ctx, ix, left, right, match_q, match_t, match_d, m)) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    return index_load(ix, {PairList{left, right, match_q, match_t, match_d, m}});
}

void sfmb200_match_index_destroy(sfmb200_match_index* ix) {
    if (!ix) return;
    std::lock_guard<std::mutex> lk(ix->ctx->mu);
    cudaSetDevice(ix->ctx->device);
    cudaStreamSynchronize(ix->ctx->stream);
    delete ix;
}

int sfmb200_find_2d3d_matches(sfmb200_match_index* ix, const uint8_t* done, int n_points, const int32_t* view_off, const int32_t* view_img,
                              const int32_t* view_feat, int64_t out_cap, int32_t* out_point, int32_t* out_feat, int64_t* out_off) {
    if (!ix) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = ix->ctx;
    const int n_img = ix->n_img;
    if (n_points < 0 || out_cap < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "negative n_points or out_cap");
    if ((n_img > 0 && !done) || !out_off || (out_cap > 0 && (!out_point || !out_feat))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (const int rc = check_views(ctx, "cloud", n_points, view_off, view_img, view_feat, ix->img_off)) return rc;
    std::vector<int32_t> views;
    for (int v = 0; v < n_img; ++v) if (!done[v]) views.push_back(v);
    const int64_t ntask = (int64_t)views.size() * n_points;
    if (ntask > INT32_MAX) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "%zu views x %d points: above 2^31 lookups in one call", views.size(), n_points);
    for (int v = 0; v <= n_img; ++v) out_off[v] = 0;
    if (ntask == 0) return SFMB200_OK;
    const int nv = view_off[n_points], nd = (int)views.size();
    const int64_t cap = std::min<int64_t>(out_cap, ntask);

    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    // pinned: the upload (views | view_off | view_img | view_feat), then what the kernels write (view starts and total, hits)
    const size_t up = Carver::pad(4 * (size_t)nd) + Carver::pad(4 * ((size_t)n_points + 1)) + 2 * Carver::pad(4 * (size_t)nv);
    const size_t pin = up + Carver::pad(4 * ((size_t)nd + 1)) + 2 * Carver::pad(4 * (size_t)cap) + 1024;
    const size_t dev = up + 2 * Carver::pad(4 * (size_t)ntask) + Carver::pad(4 * (size_t)ceil_div64(ntask, SC_CH)) + 1024;
    SFM_CUDA(ctx, ctx->pinned.reserve(pin));
    SFM_CUDA(ctx, ctx->scratch.reserve(dev));
    Carver hc(ctx->pinned.p);
    int32_t* h_views = hc.take<int32_t>(nd); int32_t* h_off = hc.take<int32_t>((size_t)n_points + 1);
    int32_t* h_img = hc.take<int32_t>(nv); int32_t* h_feat = hc.take<int32_t>(nv);
    const size_t up_len = hc.off;
    int32_t* h_vstart = hc.take<int32_t>((size_t)nd + 1);
    int32_t* h_point = hc.take<int32_t>((size_t)cap); int32_t* h_hfeat = hc.take<int32_t>((size_t)cap);
    memcpy(h_views, views.data(), 4 * (size_t)nd); memcpy(h_off, view_off, 4 * ((size_t)n_points + 1));
    if (nv) { memcpy(h_img, view_img, 4 * (size_t)nv); memcpy(h_feat, view_feat, 4 * (size_t)nv); }
    Carver dc(ctx->scratch.p);
    const int32_t* d_views = dc.take<int32_t>(nd); const int32_t* d_off = dc.take<int32_t>((size_t)n_points + 1);
    const int32_t* d_img = dc.take<int32_t>(nv); const int32_t* d_feat = dc.take<int32_t>(nv);
    int32_t* d_hit = dc.take<int32_t>((size_t)ntask); int32_t* d_flag = dc.take<int32_t>((size_t)ntask);
    int32_t* d_bsum = dc.take<int32_t>((size_t)ceil_div64(ntask, SC_CH));
    SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, ctx->pinned.p, up_len, cudaMemcpyHostToDevice, ctx->stream));
    const int nb = (int)ceil_div64(ntask, NT);
    find2d3d_kernel<<<nb, NT, 0, ctx->stream>>>((const PairRec*)ix->d_table.p, ix->pool, n_img, d_views, n_points, d_off, d_img, d_feat, d_hit,
                                                d_flag, ntask);
    SFM_LAUNCH_CHECK(ctx);
    if (const int rc = scan_excl(ctx, d_flag, (int)ntask, d_flag, d_bsum, h_vstart + nd)) return rc;
    find2d3d_write_kernel<<<nb, NT, 0, ctx->stream>>>(d_hit, d_flag, n_points, ntask, cap, h_point, h_hfeat, h_vstart);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int64_t total = h_vstart[nd];
    for (int v = 0, k = 0; v < n_img; ++v) {                           // a done view gets an empty range
        out_off[v] = k < nd ? h_vstart[k] : total;
        if (k < nd && views[k] == v) ++k;
    }
    out_off[n_img] = total;
    if (total > out_cap)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "out_cap %lld is below the %lld matches found (out_off[n_img])", (long long)out_cap, (long long)total);
    memcpy(out_point, h_point, 4 * (size_t)total); memcpy(out_feat, h_hfeat, 4 * (size_t)total);
    return SFMB200_OK;
}

int sfmb200_merge_point_cloud(sfmb200_match_index* ix, int n_exist, const float* X_exist, const int32_t* exist_off, const int32_t* exist_img,
                              const int32_t* exist_feat, int n_new, const float* X_new, const int32_t* new_off, const int32_t* new_img,
                              const int32_t* new_feat, int64_t log_cap, int8_t* outcome, int32_t* target, int32_t* log_target, int32_t* log_view,
                              int32_t* log_feat, int32_t* log_other, int32_t* log_pos, int64_t* counts) {
    if (!ix) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = ix->ctx;
    const int n_img = ix->n_img;
    if (n_exist < 0 || n_new < 0 || log_cap < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "negative n_exist, n_new or log_cap");
    if (!counts || (n_new > 0 && (!outcome || !target)) || (log_cap > 0 && (!log_target || !log_view || !log_feat)))
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if ((n_exist > 0 && !X_exist) || (n_new > 0 && !X_new)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if ((int64_t)n_exist + n_new > INT32_MAX / 4) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "too many points in one call");
    if (const int rc = check_views(ctx, "existing cloud", n_exist, exist_off, exist_img, exist_feat, ix->img_off)) return rc;
    if (const int rc = check_views(ctx, "new points", n_new, new_off, new_img, new_feat, ix->img_off)) return rc;
    const int ne = n_exist, nn = n_new, nt = ne + nn, nve = exist_off[ne], nvn = new_off[nn];
    const int64_t lbound = (int64_t)nvn * n_img;
    if (lbound > INT32_MAX / 2) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "new points' views x images above 2^30");
    counts[0] = counts[1] = counts[2] = 0;
    if (nn == 0) return SFMB200_OK;
    uint32_t H = 1024;
    while (H < 2u * (uint32_t)nt) H <<= 1;

    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const int64_t cap = std::min<int64_t>(log_cap, lbound);
    const size_t up = Carver::pad(12 * (size_t)nt) + Carver::pad(4 * ((size_t)ne + 1)) + 2 * Carver::pad(4 * (size_t)nve) +
                      Carver::pad(4 * ((size_t)nn + 1)) + 2 * Carver::pad(4 * (size_t)nvn);
    const size_t pin = up + Carver::pad((size_t)nn) + Carver::pad(4 * (size_t)nn) + 5 * Carver::pad(4 * (size_t)cap) + Carver::pad(16) + 1024;
    SFM_CUDA(ctx, ctx->pinned.reserve(pin));
    Carver hc(ctx->pinned.p);
    float* h_P = hc.take<float>(3 * (size_t)nt);
    int32_t* h_eoff = hc.take<int32_t>((size_t)ne + 1); int32_t* h_eimg = hc.take<int32_t>(nve); int32_t* h_efeat = hc.take<int32_t>(nve);
    int32_t* h_noff = hc.take<int32_t>((size_t)nn + 1); int32_t* h_nimg = hc.take<int32_t>(nvn); int32_t* h_nfeat = hc.take<int32_t>(nvn);
    const size_t up_len = hc.off;
    int8_t* h_kind = hc.take<int8_t>(nn); int32_t* h_target = hc.take<int32_t>(nn);
    Log O;
    O.target = hc.take<int32_t>((size_t)cap); O.view = hc.take<int32_t>((size_t)cap); O.feat = hc.take<int32_t>((size_t)cap);
    int32_t* h_other = hc.take<int32_t>((size_t)cap); int32_t* h_pos = hc.take<int32_t>((size_t)cap);
    O.other = log_other ? h_other : nullptr; O.pos = log_pos ? h_pos : nullptr;
    int32_t* h_tot = hc.take<int32_t>(4);                               // [0] appended, [1] log entries
    if (ne) memcpy(h_P, X_exist, 12 * (size_t)ne);
    memcpy(h_P + 3 * (size_t)ne, X_new, 12 * (size_t)nn);
    memcpy(h_eoff, exist_off, 4 * ((size_t)ne + 1)); memcpy(h_noff, new_off, 4 * ((size_t)nn + 1));
    if (nve) { memcpy(h_eimg, exist_img, 4 * (size_t)nve); memcpy(h_efeat, exist_feat, 4 * (size_t)nve); }
    if (nvn) { memcpy(h_nimg, new_img, 4 * (size_t)nvn); memcpy(h_nfeat, new_feat, 4 * (size_t)nvn); }

    const int maxn = std::max<int>((int)H, nt);
    const size_t dev = up + Carver::pad(8 * (size_t)H) + 2 * Carver::pad(4 * (size_t)H) + 5 * Carver::pad(4 * (size_t)nt) +
                       9 * Carver::pad(4 * (size_t)nn) + Carver::pad((size_t)nn) + 5 * Carver::pad(4 * (size_t)lbound) +
                       Carver::pad(4 * (size_t)ceil_div(maxn, SC_CH)) + 4096;
    SFM_CUDA(ctx, ctx->scratch.reserve(dev));
    Carver dc(ctx->scratch.p);
    const float* d_P = dc.take<float>(3 * (size_t)nt);
    const int32_t* d_eoff = dc.take<int32_t>((size_t)ne + 1); const int32_t* d_eimg = dc.take<int32_t>(nve); const int32_t* d_efeat = dc.take<int32_t>(nve);
    const int32_t* d_noff = dc.take<int32_t>((size_t)nn + 1); const int32_t* d_nimg = dc.take<int32_t>(nvn); const int32_t* d_nfeat = dc.take<int32_t>(nvn);
    uint64_t* d_tkey = dc.take<uint64_t>(H); int32_t* d_ccnt = dc.take<int32_t>(H); int32_t* d_cend = dc.take<int32_t>(H);
    int32_t* d_pslot = dc.take<int32_t>(nt); int32_t* d_cellpts = dc.take<int32_t>(nt); int* d_parent = dc.take<int>(nt);
    int32_t* d_gcnt = dc.take<int32_t>(nt); int32_t* d_gend = dc.take<int32_t>(nt);
    int32_t* d_label = dc.take<int32_t>(nn); int32_t* d_members = dc.take<int32_t>(nn); int32_t* d_bstart = dc.take<int32_t>(nn);
    int32_t* d_kind = dc.take<int32_t>(nn); int32_t* d_tnode = dc.take<int32_t>(nn); int32_t* d_lfirst = dc.take<int32_t>(nn);
    int32_t* d_lcnt = dc.take<int32_t>(nn); int32_t* d_loff = dc.take<int32_t>(nn); int32_t* d_apos = dc.take<int32_t>(nn);
    uint8_t* d_app = dc.take<uint8_t>(nn);
    Log L;
    L.target = dc.take<int32_t>((size_t)lbound); L.view = dc.take<int32_t>((size_t)lbound); L.feat = dc.take<int32_t>((size_t)lbound);
    L.other = dc.take<int32_t>((size_t)lbound); L.pos = dc.take<int32_t>((size_t)lbound);
    int32_t* d_bsum = dc.take<int32_t>((size_t)ceil_div(maxn, SC_CH));
    cudaStream_t st = ctx->stream;
    SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, ctx->pinned.p, up_len, cudaMemcpyHostToDevice, st));
    const Cloud C{d_P, d_eoff, d_eimg, d_efeat, d_noff, d_nimg, d_nfeat, ne, nn};
    const Grid G{d_tkey, d_cend, d_ccnt, d_cellpts, H - 1, 1.0 / (1.05 * (double)MERGE_POINT_DISTANCE)};   // CloudGrid's cell (host/sfm_glue.cpp)

    // grid: hashed cells, each cell's points in node order
    SFM_CUDA(ctx, cudaMemsetAsync(d_tkey, 0xff, 8 * (size_t)H, st));
    SFM_CUDA(ctx, cudaMemsetAsync(d_ccnt, 0, 4 * (size_t)H, st));
    grid_insert_kernel<<<ceil_div(nt, NT), NT, 0, st>>>(d_P, nt, G.inv, d_tkey, G.mask, d_pslot, d_ccnt);
    SFM_LAUNCH_CHECK(ctx);
    if (const int rc = scan_excl(ctx, d_ccnt, (int)H, d_cend, d_bsum, h_tot + 2)) return rc;
    grid_place_kernel<<<ceil_div(nt, NT), NT, 0, st>>>(d_pslot, nt, d_cend, d_cellpts);
    SFM_LAUNCH_CHECK(ctx);
    sort_buckets_kernel<<<ceil_div((int)H, NT), NT, 0, st>>>(d_cend, d_ccnt, (int)H, d_cellpts);
    SFM_LAUNCH_CHECK(ctx);
    // components, and each component's new points in order
    iota_kernel<<<ceil_div(nt, NT), NT, 0, st>>>(d_parent, nt);
    SFM_LAUNCH_CHECK(ctx);
    union_kernel<<<ceil_div(nn, NT), NT, 0, st>>>(C, G, d_parent);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaMemsetAsync(d_gcnt, 0, 4 * (size_t)nt, st));
    label_kernel<<<ceil_div(nn, NT), NT, 0, st>>>(ne, nn, d_parent, d_label, d_gcnt);
    SFM_LAUNCH_CHECK(ctx);
    if (const int rc = scan_excl(ctx, d_gcnt, nt, d_gend, d_bsum, h_tot + 2)) return rc;
    group_place_kernel<<<ceil_div(nn, NT), NT, 0, st>>>(d_label, nn, d_gend, d_members);
    SFM_LAUNCH_CHECK(ctx);
    sort_buckets_kernel<<<ceil_div(nt, NT), NT, 0, st>>>(d_gend, d_gcnt, nt, d_members);
    SFM_LAUNCH_CHECK(ctx);
    member_bound_kernel<<<ceil_div(nn, NT), NT, 0, st>>>(d_members, nn, d_noff, n_img, d_bstart);
    SFM_LAUNCH_CHECK(ctx);
    if (const int rc = scan_excl(ctx, d_bstart, nn, d_bstart, d_bsum, h_tot + 2)) return rc;
    // the reference's loop, component by component
    SFM_CUDA(ctx, cudaMemsetAsync(d_app, 0, (size_t)nn, st));
    resolve_kernel<<<ceil_div(nt, 128), 128, 0, st>>>(C, G, (const PairRec*)ix->d_table.p, ix->pool, n_img, d_gend, d_gcnt, d_members, d_bstart,
                                                      d_app, d_kind, d_tnode, d_lfirst, d_lcnt, L);
    SFM_LAUNCH_CHECK(ctx);
    // appended points' cloud indices and the log's order (new point by new point)
    appended_flags_kernel<<<ceil_div(nn, NT), NT, 0, st>>>(d_app, nn, d_apos);
    SFM_LAUNCH_CHECK(ctx);
    if (const int rc = scan_excl(ctx, d_apos, nn, d_apos, d_bsum, h_tot + 0)) return rc;
    if (const int rc = scan_excl(ctx, d_lcnt, nn, d_loff, d_bsum, h_tot + 1)) return rc;
    merge_write_kernel<<<ceil_div(nn, NT), NT, 0, st>>>(ne, nn, d_kind, d_tnode, d_apos, d_lfirst, d_lcnt, d_loff, L, cap, h_kind, h_target, O);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaStreamSynchronize(st));
    const int64_t n_log = h_tot[1];
    counts[0] = h_tot[0];
    counts[2] = n_log;
    int64_t merged = 0;
    for (int i = 0; i < nn; ++i) merged += h_kind[i] == SFMB200_MERGE_MERGED;
    counts[1] = merged;
    if (n_log > log_cap)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "log_cap %lld is below the %lld assignments of this merge (counts[2])", (long long)log_cap, (long long)n_log);
    memcpy(outcome, h_kind, (size_t)nn); memcpy(target, h_target, 4 * (size_t)nn);
    memcpy(log_target, O.target, 4 * (size_t)n_log); memcpy(log_view, O.view, 4 * (size_t)n_log); memcpy(log_feat, O.feat, 4 * (size_t)n_log);
    if (log_other) memcpy(log_other, h_other, 4 * (size_t)n_log);
    if (log_pos) memcpy(log_pos, h_pos, 4 * (size_t)n_log);
    return SFMB200_OK;
}

}  // extern "C"
