// orb.cu -- SURVEY.md section 8 row f-3: ORB extraction, the step before matching.
//
// Replaces SfM2DFeatureUtilities::extractFeatures (SfM2DFeatureUtilities.cpp:46-51) = `ORB::create(5000)->detectAndCompute(image,
// noArray(), keyPoints, descriptors)` (:39, :48) for one image or for all images of SfM::extractFeatures (SfM.cpp:141-154) in one
// call.  Results are bit-identical to OpenCV's: key points (pt, size, angle, response, octave) in OpenCV's output order and the
// 256-bit descriptors (tests/test_gpu_orb.py compares with cv2 on real and synthetic images and with oracle/orb_oracle.py stage by stage).
//
// Work split.  Everything that touches pixels runs on the GPU: grey conversion, the 8-level INTER_LINEAR_EXACT pyramid, FAST-9/16 scores
// of every pyramid pixel, 3x3 non-maximum suppression + border filter + ORDERED compaction (raster order inside a level, the order
// cv::FAST emits), Harris responses, intensity-centroid angles, the float separable Gaussian, steered BRIEF.  The two
// `KeyPointsFilter::retainBest` selections stay on the host ON PURPOSE: their result ORDER is whatever libstdc++'s std::nth_element +
// std::partition leave behind, and every later stage (and the matcher's trainIdx) inherits that order -- running the same two
// algorithms on 8-byte (response, index) records reproduces it exactly and costs ~0.1 ms per image.
// All kernels carry the image index in blockIdx.z, the tile list or the record and look up that image's layout (sizes and arena
// offsets, orb_groups.h) in a device table, so a group of images of any sizes shares every launch and every host<->device round trip
// (3 per group).  The images come from host memory (staged and uploaded here) or are already on the device (sfmb200_decode_jpeg_extract_orb).
//
// Integer / byte work, HBM- and latency-bound (2.6 MB of pyramid per 1024x768 image): no tensor cores involved.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <map>
#include <memory>

#include "common.cuh"
#include "orb_groups.h"
#include "orb_math.cuh"
#define ORB_PATTERN_DECL __device__
#include "orb_pattern.h"

namespace {

constexpr int ORB_EDGE = 31;          // edgeThreshold
constexpr int ORB_FAST_T = 20;        // fastThreshold

// resize(INTER_LINEAR_EXACT) tap tables: for destination index d, the two source indices and the weight (1/256) of the second one.
void linear_exact_taps(int src, int dst, int32_t* i0, int32_t* i1, int32_t* a) {
    const double scale = (double)src / (double)dst;
    for (int d = 0; d < dst; d++) {
        const double f = scale * ((double)d + 0.5) - 0.5;
        const int i = (int)std::floor(f);
        int w = (int)std::nearbyint((f - (double)i) * 256.0);
        int lo = i, hi = i + 1;
        if (i < 0) { lo = hi = 0; w = 0; }
        if (i >= src - 1) { lo = hi = src - 1; w = 0; }
        i0[d] = lo; i1[d] = hi; a[d] = w;
    }
}

// KeyPointsFilter::retainBest on (response, index) records: same std algorithms, same comparator results, hence the same permutation.
struct Rec { float response; int32_t idx; };
struct RecGreater { bool operator()(const Rec& a, const Rec& b) const { return a.response > b.response; } };
struct RecAtLeast { float v; bool operator()(const Rec& k) const { return k.response >= v; } };
void retain_best(std::vector<Rec>& k, int n_points) {
    if (n_points >= 0 && k.size() > (size_t)n_points) {
        if (n_points == 0) { k.clear(); return; }
        std::nth_element(k.begin(), k.begin() + n_points - 1, k.end(), RecGreater());
        const float ambiguous = k[n_points - 1].response;
        auto new_end = std::partition(k.begin() + n_points, k.end(), RecAtLeast{ambiguous});
        k.resize(new_end - k.begin());
    }
}

// ---------------------------------------------------------------------------------------------------- kernels
// Tile lists of the FAST and blur kernels: one 32-bit word per tile row of a group, image slot << 16 | level << 13 | first row / 16.
// The grid is flat: block b works on tile b / xblocks and 32- or 64-pixel column b % xblocks, with xblocks from the group's widest image.
__host__ __device__ __forceinline__ uint32_t tile_word(int slot, int l, int y0) { return (uint32_t)slot << 16 | (uint32_t)l << 13 | (uint32_t)(y0 >> 4); }

// grid = (columns of the widest image / 256, rows of the tallest, images); Ls = the layouts of the launch's images
__global__ void __launch_bounds__(256) orb_gray_kernel(const OrbLayout* __restrict__ Ls, uint8_t* __restrict__ pyr) {
    const OrbLayout& L = Ls[blockIdx.z];
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, w = L.lv[0].w;
    if (x >= w || y >= L.lv[0].h) return;
    const uint8_t* p = L.src + (size_t)y * L.src_stride + 3 * x;
    pyr[L.pix0 + (size_t)y * w + x] = (uint8_t)orbm::gray_from_bgr(p[0], p[1], p[2]);
}

// level l from level l - 1; taps (x: i0,i1,a [dw each]; y: i0,i1,a [dh each]) at the level's offset in the group's table
__global__ void __launch_bounds__(256) orb_resize_kernel(const OrbLayout* __restrict__ Ls, uint8_t* pyr, int l, const int32_t* __restrict__ taps_all) {
    const OrbLayout& L = Ls[blockIdx.z];
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    const OrbLevel& d = L.lv[l];
    const int dw = d.w, dh = d.h;
    if (x >= dw || y >= dh) return;
    const int sw = L.lv[l - 1].w;
    const int32_t* taps = taps_all + d.taps;
    const int x0 = taps[x], x1 = taps[dw + x], ax = taps[2 * dw + x];
    const int32_t* ty = taps + 3 * dw;
    const int y0 = ty[y], y1 = ty[dh + y], ay = ty[2 * dh + y];
    const uint8_t* s = pyr + L.pix0 + L.lv[l - 1].off;
    const int v = orbm::resize_linear_exact(s[(size_t)y0 * sw + x0], s[(size_t)y0 * sw + x1], s[(size_t)y1 * sw + x0], s[(size_t)y1 * sw + x1], ax, ay);
    pyr[L.pix0 + d.off + (size_t)y * dw + x] = (uint8_t)v;
}

// FAST-9/16: the four compass points decide whether a position can be a corner at all (9-18 % of the pixels of a photograph pass, but
// half of all 32-pixel rows hold at least one such pixel), so a tile first collects the positions that pass in a shared list and then
// spends the 12 remaining loads and the 9-arc network on a DENSE list instead of on half-empty warps.
__device__ __forceinline__ bool fast_candidate(const uint8_t* __restrict__ I, int w, int h, int x, int y) {
    if (x < 3 || x >= w - 3 || y < 3 || y >= h - 3) return false;
    const uint8_t* c = I + (size_t)y * w + x;
    return orbm::fast9_may_be_corner(c[0], c[3 * w], c[3], c[-3 * w], c[-3], ORB_FAST_T);
}
__device__ __forceinline__ int fast_full(const uint8_t* __restrict__ I, int w, int x, int y) {
    const uint8_t* c = I + (size_t)y * w + x;
    int p[16];
    p[0] = c[3 * w];       p[1] = c[3 * w + 1];   p[2] = c[2 * w + 2];   p[3] = c[w + 3];
    p[4] = c[3];           p[5] = c[-w + 3];      p[6] = c[-2 * w + 2];  p[7] = c[-3 * w + 1];
    p[8] = c[-3 * w];      p[9] = c[-3 * w - 1];  p[10] = c[-2 * w - 2]; p[11] = c[-w - 3];
    p[12] = c[-3];         p[13] = c[w - 3];      p[14] = c[2 * w - 2];  p[15] = c[3 * w - 1];
    return orbm::fast9_score(c[0], p, ORB_FAST_T);
}

// FAST scores of a 32 x 32 tile (+1 halo) in shared memory -> score map; 3x3 non-maximum suppression (fast.cpp: strictly greater than the 8
// neighbours) + KeyPointsFilter::runByImageBorder(edgeThreshold) -> one 32-bit survivor mask per (row, 32-pixel word) and the number of
// survivors per pyramid row (integer atomics: order-independent).  The tile is 32 rows high so that the dense candidate list (~150 of
// 1156 positions) fills the CTA's 8 warps in the scoring phase -- with 8-row tiles two warps scored while six waited at the barrier
// (ncu: barrier = top stall) -- and the halo costs 13 % instead of 33 %.
// grid = xblocks (survivor words per row of the widest image) x tile rows of the launch's images, block = (32, 8): thread (x, y) owns
// rows y, y+8, y+16, y+24.
constexpr int FT_W = 32, FT_H = 32, FT_TY = 8, FT_N = (FT_W + 2) * (FT_H + 2);
__global__ void __launch_bounds__(FT_W * FT_TY) orb_fast_nms_kernel(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ score, uint32_t* __restrict__ mask,
                                                                     int32_t* __restrict__ row_cnt, const OrbLayout* __restrict__ Ls,
                                                                     const uint32_t* __restrict__ tiles, int xblocks) {
    __shared__ uint8_t sc[FT_H + 2][FT_W + 2 + 2];
    __shared__ uint16_t list[FT_N];
    __shared__ int nlist;
    const uint32_t tile = tiles[blockIdx.x / xblocks];
    const int bx = blockIdx.x % xblocks, l = (tile >> 13) & 7, y0 = (int)(tile & 0x1FFF) << 4, x0 = bx * FT_W;
    const OrbLayout& L = Ls[tile >> 16];
    if (bx >= L.chunks) return;                      // past this image's own words
    const int w = L.lv[l].w, h = L.lv[l].h, row0 = L.lv[l].row0, chunks = L.chunks;
    uint32_t* M = mask + L.mask0;
    if (x0 >= w) {                                   // words beyond this level's width: the scatter walks all `chunks` words of a row
        if (threadIdx.x == 0)
            for (int ry = threadIdx.y; ry < FT_H && y0 + ry < h; ry += FT_TY) M[(size_t)(row0 + y0 + ry) * chunks + bx] = 0u;
        return;
    }
    const uint8_t* I = pyr + L.pix0 + L.lv[l].off;
    const int tid = threadIdx.y * FT_W + threadIdx.x;
    if (tid == 0) nlist = 0;
    __syncthreads();
    for (int t = tid; t < FT_N; t += FT_W * FT_TY) {
        const int tx = t % (FT_W + 2), ty = t / (FT_W + 2);
        sc[ty][tx] = 0;
        if (fast_candidate(I, w, h, x0 - 1 + tx, y0 - 1 + ty)) list[atomicAdd(&nlist, 1)] = (uint16_t)t;
    }
    __syncthreads();
    for (int i = tid; i < nlist; i += FT_W * FT_TY) {
        const int t = list[i], tx = t % (FT_W + 2), ty = t / (FT_W + 2);
        sc[ty][tx] = (uint8_t)fast_full(I, w, x0 - 1 + tx, y0 - 1 + ty);
    }
    __syncthreads();
    const int x = x0 + threadIdx.x;
    uint8_t* S = score + L.pix0 + L.lv[l].off;
#pragma unroll
    for (int ry = threadIdx.y; ry < FT_H; ry += FT_TY) {
        const int y = y0 + ry;
        const int s = sc[ry + 1][threadIdx.x + 1];
        bool keep = false;
        if (x < w && y < h) {
            S[(size_t)y * w + x] = (uint8_t)s;
            if (s && x >= ORB_EDGE && x < w - ORB_EDGE && y >= ORB_EDGE && y < h - ORB_EDGE) {
                const uint8_t* r0 = &sc[ry][threadIdx.x]; const uint8_t* r1 = r0 + (FT_W + 4); const uint8_t* r2 = r1 + (FT_W + 4);
                keep = s > r0[0] && s > r0[1] && s > r0[2] && s > r1[0] && s > r1[2] && s > r2[0] && s > r2[1] && s > r2[2];
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (threadIdx.x == 0 && y < h) {
            const int row = row0 + y;
            M[(size_t)row * chunks + bx] = m;
            if (m) atomicAdd(&row_cnt[L.cnt0 + row], __popc(m));
        }
    }
}

// Exclusive scan of the survivors per pyramid row of one image (one CTA per image); start of every level and the total.
__global__ void __launch_bounds__(1024) orb_scan_kernel(const int32_t* __restrict__ row_cnt, int32_t* __restrict__ row_off, int32_t* __restrict__ lvl_start,
                                                        const OrbLayout* __restrict__ Ls) {
    __shared__ int warp_sum[32];
    __shared__ int carry;
    const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const OrbLayout& L = Ls[img];
    const int total_rows = L.total_rows;
    const int32_t* c = row_cnt + L.cnt0; int32_t* o = row_off + L.cnt0;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < total_rows; base += 1024) {
        const int r = base + tid;
        const int v = r < total_rows ? c[r] : 0;
        int s = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += t; }
        if (lane == 31) warp_sum[wid] = s;
        __syncthreads();
        if (wid == 0) {
            int t = warp_sum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, t, d); if (lane >= d) t += u; }
            warp_sum[lane] = t;
        }
        __syncthreads();
        const int before = carry + (wid ? warp_sum[wid - 1] : 0) + s - v;
        if (r < total_rows) o[r] = before;
        __syncthreads();
        if (tid == 1023) carry = before + v;
        __syncthreads();
    }
    if (tid == 0) o[total_rows] = carry;
    __syncthreads();
    if (tid <= ORB_LEVELS) lvl_start[img * 16 + tid] = (tid < ORB_LEVELS && L.lv[tid].h > 0) ? o[L.lv[tid].row0] : carry;
}

// Ordered scatter: one warp per pyramid row -> candidates (x | y << 16, score | level << 16), raster order inside a level (the order cv::FAST
// emits), levels back to back.  grid = (rows of the image with the most pyramid rows / 8, 1, images)
__global__ void __launch_bounds__(256) orb_scatter_kernel(const uint32_t* __restrict__ mask, const uint8_t* __restrict__ score, const int32_t* __restrict__ row_off,
                                                           const OrbLayout* __restrict__ Ls, uint2* __restrict__ cand) {
    const OrbLayout& L = Ls[blockIdx.z];
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (row >= L.total_rows) return;
    int l = 0;
#pragma unroll
    for (int i = 1; i < ORB_LEVELS; i++) l += (L.lv[i].h > 0 && row >= L.lv[i].row0) ? 1 : 0;
    const int w = L.lv[l].w, y = row - L.lv[l].row0, chunks = L.chunks, cand_cap = L.cand_cap;
    const uint8_t* sc = score + L.pix0 + L.lv[l].off + (size_t)y * w;
    int pos = row_off[L.cnt0 + row];
    uint2* out = cand + L.cand0;
    const uint32_t* M = mask + L.mask0 + (size_t)row * chunks;
    for (int j0 = 0; j0 < chunks; j0 += 32) {
        const int j = j0 + lane;
        unsigned m = j < chunks ? M[j] : 0u;
        const int c = __popc(m);
        int incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
        int at = pos + incl - c;
        while (m) {
            const int bit = __ffs(m) - 1; m &= m - 1;
            const int x = j * 32 + bit;
            if (at < cand_cap) out[at] = make_uint2((unsigned)x | ((unsigned)y << 16), (unsigned)sc[x] | ((unsigned)l << 16));
            at++;
        }
        pos += __shfl_sync(0xffffffffu, incl, 31);
    }
}

// Harris response of selected candidates: one warp per record {x | y << 16, level | img << 8}.
__global__ void __launch_bounds__(256) orb_harris_kernel(const uint8_t* __restrict__ pyr, const OrbLayout* __restrict__ Ls, const uint2* __restrict__ sel, int n,
                                                          float* __restrict__ response) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n) return;
    const uint2 r = sel[i];
    const int x = r.x & 0xFFFF, y = r.x >> 16, l = r.y & 0xFF, img = r.y >> 8;
    const OrbLayout& L = Ls[img];
    const int w = L.lv[l].w;
    const uint8_t* I = pyr + L.pix0 + L.lv[l].off;
    int a = 0, b = 0, c = 0;
    for (int k = lane; k < 49; k += 32) {
        const uint8_t* p = I + (size_t)(y - 3 + k / 7) * w + (x - 3 + k % 7);
        const int ix = ((int)p[1] - (int)p[-1]) * 2 + ((int)p[-w + 1] - (int)p[-w - 1]) + ((int)p[w + 1] - (int)p[w - 1]);
        const int iy = ((int)p[w] - (int)p[-w]) * 2 + ((int)p[w - 1] - (int)p[-w - 1]) + ((int)p[w + 1] - (int)p[-w + 1]);
        a += ix * ix; b += iy * iy; c += ix * iy;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, d); b += __shfl_xor_sync(0xffffffffu, b, d); c += __shfl_xor_sync(0xffffffffu, c, d); }
    if (lane == 0) response[i] = orbm::harris_response(a, b, c);
}

// Float separable Gaussian of every level (BORDER_REFLECT_101).  Tile 64 x 16 per CTA; grid = xblocks (64-pixel columns of the widest
// image) x tile rows (16 rows each) of the launch's images.
constexpr int BT_W = 64, BT_H = 16;
__device__ __forceinline__ int reflect101(int i, int n) { i = i < 0 ? -i : i; return i >= n ? 2 * n - 2 - i : i; }
__global__ void __launch_bounds__(256) orb_blur_kernel(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ blur, const OrbLayout* __restrict__ Ls,
                                                        const uint32_t* __restrict__ tiles, int xblocks) {
    __shared__ float R[BT_H + 6][BT_W];
    const uint32_t tile = tiles[blockIdx.x / xblocks];
    const int l = (tile >> 13) & 7, y0 = (int)(tile & 0x1FFF) << 4, x0 = (blockIdx.x % xblocks) * BT_W;
    const OrbLayout& L = Ls[tile >> 16];
    const int w = L.lv[l].w, h = L.lv[l].h;
    if (x0 >= w) return;
    const uint8_t* I = pyr + L.pix0 + L.lv[l].off;
    uint8_t* O = blur + L.pix0 + L.lv[l].off;
    if (w < 4 || h < 4) {                               // too small to reflect: copy (such a level cannot hold a key point anyway)
        for (int t = threadIdx.x; t < BT_W * BT_H; t += 256) {
            const int x = x0 + t % BT_W, y = y0 + t / BT_W;
            if (x < w && y < h) O[(size_t)y * w + x] = I[(size_t)y * w + x];
        }
        return;
    }
    for (int t = threadIdx.x; t < BT_W * (BT_H + 6); t += 256) {
        const int tx = t % BT_W, ty = t / BT_W, x = x0 + tx, y = reflect101(y0 + ty - 3, h);
        float v = 0.f;
        if (x < w && y0 + ty - 3 < h + 3) {
            const uint8_t* row = I + (size_t)y * w;
            int p[7];
#pragma unroll
            for (int k = 0; k < 7; k++) p[k] = row[reflect101(x + k - 3, w)];
            v = orbm::blur_row(p);
        }
        R[ty][tx] = v;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < BT_W * BT_H; t += 256) {
        const int tx = t % BT_W, ty = t / BT_W, x = x0 + tx, y = y0 + ty;
        if (x < w && y < h) {
            float r[7];
#pragma unroll
            for (int k = 0; k < 7; k++) r[k] = R[ty + k][tx];
            O[(size_t)y * w + x] = (uint8_t)orbm::blur_col(r);
        }
    }
}

// cv::KeyPoint, 28 bytes: the shim can copy these straight into std::vector<cv::KeyPoint>
struct KeyPointOut { float x, y, size, angle, response; int32_t octave, class_id; };

// ICAngles + computeOrbDescriptors + the final `pt *= scale`: one warp per key point record {x | y << 16, level | img << 8}.
__global__ void __launch_bounds__(256) orb_describe_kernel(const uint8_t* __restrict__ pyr, const uint8_t* __restrict__ blur, const OrbLayout* __restrict__ Ls,
                                                            const uint2* __restrict__ sel, const float* __restrict__ response, int n,
                                                            KeyPointOut* __restrict__ kp, uint8_t* __restrict__ desc) {
    __shared__ signed char pat[1024];
    for (int t = threadIdx.x; t < 1024; t += blockDim.x) pat[t] = ORB_BIT_PATTERN_31[t];
    __syncthreads();
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n) return;
    const uint2 r = sel[i];
    const int x = r.x & 0xFFFF, y = r.x >> 16, l = r.y & 0xFF, img = r.y >> 8;
    const OrbLayout& L = Ls[img];
    const int w = L.lv[l].w;
    const uint8_t* I = pyr + L.pix0 + L.lv[l].off;
    // intensity centroid over the circular patch of radius 15: lane = row v + 15
    int m10 = 0, m01 = 0;
    if (lane < 31) {
        const int v = lane - 15, u = orbm::umax15(v < 0 ? -v : v);
        const uint8_t* row = I + (size_t)(y + v) * w + x;
        int sum = 0;
        for (int k = -u; k <= u; k++) { const int p = row[k]; sum += p; m10 += k * p; }
        m01 = v * sum;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) { m10 += __shfl_xor_sync(0xffffffffu, m10, d); m01 += __shfl_xor_sync(0xffffffffu, m01, d); }
    const float angle = orbm::fast_atan2((float)m01, (float)m10);
    const float scale = L.lv[l].scale, inv = L.lv[l].inv_scale;
    const float px = orbm::mul((float)x, scale), py = orbm::mul((float)y, scale);            // keypoints[i].pt *= scale
    if (lane == 0) {
        KeyPointOut o; o.x = px; o.y = py; o.size = orbm::mul(31.0f, scale); o.angle = angle; o.response = response[i]; o.octave = l; o.class_id = -1;
        kp[i] = o;
    }
    // steered BRIEF on the blurred level, centre = (cvRound(pt.x * (1/scale)), cvRound(pt.y * (1/scale))); lane = descriptor byte
    const int cx = orbm::round_even(orbm::mul(px, inv)), cy = orbm::round_even(orbm::mul(py, inv));
    float a, b;
    orbm::angle_to_cs(angle, &a, &b);
    const uint8_t* C = blur + L.pix0 + L.lv[l].off + (size_t)cy * w + cx;
    unsigned byte = 0;
#pragma unroll
    for (int bit = 0; bit < 8; bit++) {
        const signed char* q = pat + (lane * 8 + bit) * 4;
        const int t0 = C[orbm::rot_y(q[0], q[1], a, b) * w + orbm::rot_x(q[0], q[1], a, b)];
        const int t1 = C[orbm::rot_y(q[2], q[3], a, b) * w + orbm::rot_x(q[2], q[3], a, b)];
        byte |= (unsigned)(t0 < t1) << bit;
    }
    desc[(size_t)i * 32 + lane] = (uint8_t)byte;
}

// ---------------------------------------------------------------------------------------------------- host driver
// One image size: its layout (arena offsets zero), its resize taps (per level l >= 1: x taps (3 * w_l) then y taps (3 * h_l); lv[l].taps
// counts from the start of this vector) and the tile rows of the blur (BT_H rows) and FAST (FT_H rows) kernels as tile words of slot 0.
struct OrbPlan {
    OrbLayout L;
    std::vector<int32_t> taps;
    std::vector<uint32_t> blur_tiles, fast_tiles;
};

void make_plan(int w, int h, int nfeatures, OrbPlan& P) {
    make_layout(w, h, nfeatures, P.L);
    P.taps.clear();
    for (int l = 0; l < ORB_LEVELS; l++) {
        OrbLevel& d = P.L.lv[l];
        d.taps = (int)P.taps.size();
        if (l == 0 || d.w == 0) continue;
        const OrbLevel& s = P.L.lv[l - 1];
        const size_t at = P.taps.size();
        P.taps.resize(at + 3 * (size_t)d.w + 3 * (size_t)d.h);
        int32_t* t = P.taps.data() + at;
        linear_exact_taps(s.w, d.w, t, t + d.w, t + 2 * d.w);
        t += 3 * d.w;
        linear_exact_taps(s.h, d.h, t, t + d.h, t + 2 * d.h);
    }
    P.blur_tiles.clear(); P.fast_tiles.clear();
    for (int l = 0; l < ORB_LEVELS; l++) {
        for (int y = 0; y < P.L.lv[l].h; y += BT_H) P.blur_tiles.push_back(tile_word(0, l, y));
        for (int y = 0; y < P.L.lv[l].h; y += FT_H) P.fast_tiles.push_back(tile_word(0, l, y));
    }
}

// The images of one call: host images (staged in pinned memory and uploaded here, all of one size) or B,G,R images that are already on
// the device (packed rows, any sizes).
struct OrbInput {
    const uint8_t* const* host = nullptr; int channels = 3; size_t row_stride = 0;
    const uint8_t* const* dev = nullptr;
};

// One group of images: the layouts of its slots with their arena offsets, its tables and the sizes of its arenas.
struct OrbGroup {
    int i0 = 0, nb = 0;                                   // first image of the call, images
    std::vector<OrbLayout> L;
    std::vector<int32_t> taps;                            // the taps of every distinct size of the group, once
    std::vector<uint32_t> blur_tiles, fast_tiles;
    std::vector<int> blur_at, fast_at;                    // first tile of every slot, then the total
    std::vector<size_t> raw0, stage0;                     // slot's B,G,R upload in the raw arena / its host image in the pinned staging
    size_t raw = 0, stage = 0, pix = 0, mask = 0, cnt = 0, cand = 0;    // bytes, bytes, bytes, mask words, row counters, candidates
};

void make_group(const std::vector<const OrbPlan*>& plan_of, int i0, int i1, const OrbInput& in, OrbGroup& G) {
    G = OrbGroup{};
    G.i0 = i0; G.nb = i1 - i0;
    std::vector<std::pair<const OrbPlan*, int>> taps_at;
    for (int s = 0; s < G.nb; s++) {
        const OrbPlan& P = *plan_of[i0 + s];
        int t0 = -1;
        for (auto& pt : taps_at) if (pt.first == &P) t0 = pt.second;
        if (t0 < 0) { t0 = (int)G.taps.size(); taps_at.emplace_back(&P, t0); G.taps.insert(G.taps.end(), P.taps.begin(), P.taps.end()); }
        OrbLayout L = P.L;
        for (int l = 0; l < ORB_LEVELS; l++) L.lv[l].taps += t0;
        const size_t px = (size_t)L.lv[0].w * L.lv[0].h;
        L.pix0 = G.pix; G.pix += (size_t)L.slab;
        L.mask0 = G.mask; G.mask += (size_t)L.ncnt;
        L.cnt0 = G.cnt; G.cnt += (size_t)L.total_rows + 1;
        L.cand0 = G.cand; G.cand += (size_t)L.cand_cap;
        L.src_stride = 3 * L.lv[0].w;
        G.raw0.push_back(G.raw); G.raw += in.host && in.channels == 3 ? 3 * px : 0;
        G.stage0.push_back(G.stage); G.stage += in.host ? px * in.channels : 0;
        G.L.push_back(L);
        G.blur_at.push_back((int)G.blur_tiles.size());
        for (uint32_t t : P.blur_tiles) G.blur_tiles.push_back(t | (uint32_t)s << 16);
        G.fast_at.push_back((int)G.fast_tiles.size());
        for (uint32_t t : P.fast_tiles) G.fast_tiles.push_back(t | (uint32_t)s << 16);
    }
    G.blur_at.push_back((int)G.blur_tiles.size()); G.fast_at.push_back((int)G.fast_tiles.size());
}

// Device pointers of a group, carved in this order from ctx->orb_dev; the tables come first and mirror their pinned staging.
struct OrbDev {
    OrbLayout* L; int32_t* taps; uint32_t *blur_tiles, *fast_tiles;
    uint8_t *raw, *pyr, *blur, *score; uint32_t* mask; int32_t *rowoff, *rowcnt, *lvl; uint2* cand;
};
size_t carve_tables(Carver& c, const OrbGroup& G, OrbDev& D) {
    D.L = c.take<OrbLayout>(G.L.size());
    D.taps = c.take<int32_t>(G.taps.size() + 4);
    D.blur_tiles = c.take<uint32_t>(G.blur_tiles.size() + 4); D.fast_tiles = c.take<uint32_t>(G.fast_tiles.size() + 4);
    return c.off;
}
size_t carve(Carver& c, const OrbGroup& G, OrbDev& D) {
    carve_tables(c, G, D);
    D.raw = c.take<uint8_t>(G.raw);
    D.pyr = c.take<uint8_t>(G.pix); D.blur = c.take<uint8_t>(G.pix); D.score = c.take<uint8_t>(G.pix);
    D.mask = c.take<uint32_t>(G.mask); D.rowoff = c.take<int32_t>(G.cnt); D.rowcnt = c.take<int32_t>(G.cnt);
    D.lvl = c.take<int32_t>(16 * (size_t)G.nb);
    D.cand = c.take<uint2>(G.cand);
    return c.off;
}

inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// Grey, pyramid, blur (side stream), FAST + suppression of slots [s0, s0 + n) of a group: no host involvement.
int orb_detect(sfmb200_ctx* ctx, const OrbGroup& G, const OrbDev& D, int s0, int n, bool grey_from_bgr) {
    cudaStream_t st = ctx->stream;
    int maxw = 0, maxh = 0, maxchunks = 0;
    for (int s = s0; s < s0 + n; s++) {
        maxw = std::max(maxw, G.L[s].lv[0].w); maxh = std::max(maxh, G.L[s].lv[0].h); maxchunks = std::max(maxchunks, G.L[s].chunks);
    }
    if (grey_from_bgr) {
        orb_gray_kernel<<<dim3(ceil_div(maxw, 256), maxh, n), 256, 0, st>>>(D.L + s0, D.pyr);
        SFM_LAUNCH_CHECK(ctx);
    }
    for (int l = 1; l < ORB_LEVELS; l++) {
        int dw = 0, dh = 0;
        for (int s = s0; s < s0 + n; s++) { dw = std::max(dw, G.L[s].lv[l].w); dh = std::max(dh, G.L[s].lv[l].h); }
        if (dw == 0) break;
        orb_resize_kernel<<<dim3(ceil_div(dw, 256), dh, n), 256, 0, st>>>(D.L + s0, D.pyr, l, D.taps);
        SFM_LAUNCH_CHECK(ctx);
    }
    SFM_CUDA(ctx, cudaEventRecord(ctx->orb_ev[0], st));
    SFM_CUDA(ctx, cudaStreamWaitEvent(ctx->orb_stream, ctx->orb_ev[0], 0));
    const int xb = ceil_div(maxw, BT_W);
    const int64_t nbt = G.blur_at[s0 + n] - G.blur_at[s0], nft = G.fast_at[s0 + n] - G.fast_at[s0];
    orb_blur_kernel<<<(unsigned)(nbt * xb), 256, 0, ctx->orb_stream>>>(D.pyr, D.blur, D.L, D.blur_tiles + G.blur_at[s0], xb);
    SFM_LAUNCH_CHECK(ctx);
    orb_fast_nms_kernel<<<(unsigned)(nft * maxchunks), dim3(FT_W, FT_TY), 0, st>>>(D.pyr, D.score, D.mask, D.rowcnt, D.L, D.fast_tiles + G.fast_at[s0], maxchunks);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

// Input stage for host images: staging + upload, pipelined against detection.  The pool packs quarter images into pinned memory IN
// IMAGE ORDER and every thread sends its piece off itself on the upload stream (a pageable cudaMemcpy would pack and copy serially on one
// thread); whoever enqueues the last piece of an image records that image's event.  Detection runs per GROUP of images on the main
// stream as soon as the group's images have landed, i.e. under the DMA of the following groups: the call is PCIe-bound.  Only worth it
// for large batches (measured: 50 images 11.5 -> 9.9 ms, but 7 images 2.8 -> 3.5 ms -- 4x the launches on quarter-size grids and 28 small
// copies): small batches send whole images and run detection once.
int orb_input_host(sfmb200_ctx* ctx, const OrbGroup& G, const OrbDev& D, const OrbInput& in) {
    const int nb = G.nb, dev = ctx->device, channels = in.channels;
    const bool pipelined = nb >= 16;
    const int PIECES = pipelined ? 4 : 1;
    while ((int)ctx->orb_img_ev.size() < nb) {
        cudaEvent_t ev = nullptr;
        SFM_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        ctx->orb_img_ev.push_back(ev);
    }
    std::unique_ptr<std::atomic<int>[]> pieces_done(new std::atomic<int>[nb]);
    for (int s = 0; s < nb; s++) pieces_done[s].store(0);
    std::atomic<int> task_err{0};
    uint8_t* h_img = (uint8_t*)ctx->orb_pin_img.p;
    cudaStream_t up = ctx->orb_up;
    SFM_CUDA(ctx, cudaEventRecord(ctx->orb_ev[0], ctx->stream));         // the previous group's kernels have read the buffers the uploads overwrite
    SFM_CUDA(ctx, cudaStreamWaitEvent(up, ctx->orb_ev[0], 0));
    host_pool(ctx).parallel_for(nb * PIECES, [&](int t) {
        cudaSetDevice(dev);
        const int s = t / PIECES, c = t % PIECES;
        const OrbLayout& L = G.L[s];
        const int w = L.lv[0].w, h = L.lv[0].h;
        const int y0 = (int)((int64_t)h * c / PIECES), y1 = (int)((int64_t)h * (c + 1) / PIECES);
        const size_t rb = (size_t)w * channels, off = (size_t)y0 * rb, bytes = (size_t)(y1 - y0) * rb;
        uint8_t* dst = h_img + G.stage0[s] + off; const uint8_t* src = in.host[G.i0 + s] + (size_t)y0 * in.row_stride;
        if (in.row_stride == rb) memcpy(dst, src, bytes);
        else for (int y = 0; y < y1 - y0; y++) memcpy(dst + (size_t)y * rb, src + (size_t)y * in.row_stride, rb);
        uint8_t* d = (channels == 1 ? D.pyr + L.pix0 : D.raw + G.raw0[s]) + off;
        if (bytes && cudaMemcpyAsync(d, dst, bytes, cudaMemcpyHostToDevice, up) != cudaSuccess) task_err.store(1);
        if (pieces_done[s].fetch_add(1) + 1 == PIECES && cudaEventRecord(ctx->orb_img_ev[s], up) != cudaSuccess) task_err.store(1);
    });
    if (task_err.load()) return sfmb200_fail(ctx, SFMB200_ERR_CUDA, "image upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    const int groups = pipelined ? 4 : 1, gsz = ceil_div(nb, groups);
    for (int s0 = 0; s0 < nb; s0 += gsz) {
        const int n = std::min(gsz, nb - s0);
        for (int s = s0; s < s0 + n; s++) SFM_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->orb_img_ev[s], 0));
        if (int rc = orb_detect(ctx, G, D, s0, n, channels == 3)) return rc;
    }
    return SFMB200_OK;
}

// The rest of the stage, whatever the input: ordered compaction, the three host round trips with the two retainBest selections,
// describe, copy-out of the group's key points and descriptors.
int orb_finish(sfmb200_ctx* ctx, const OrbGroup& G, const OrbDev& D, int cap, KeyPointOut* kp_out, uint8_t* desc_out, int32_t* n_out,
               std::vector<std::vector<Rec>>& task, double t0) {
    cudaStream_t st = ctx->stream;
    HostPool& pool = host_pool(ctx);
    double* tm = ctx->orb_ms;
    const int nb = G.nb, i0 = G.i0;
    int max_rows = 0;
    for (const OrbLayout& L : G.L) max_rows = std::max(max_rows, L.total_rows);
    SFM_CUDA(ctx, cudaEventRecord(ctx->orb_ev[1], ctx->orb_stream));
    orb_scan_kernel<<<nb, 1024, 0, st>>>(D.rowcnt, D.rowoff, D.lvl, D.L); SFM_LAUNCH_CHECK(ctx);
    orb_scatter_kernel<<<dim3(ceil_div(max_rows * 32, 256), 1, nb), 256, 0, st>>>(D.mask, D.score, D.rowoff, D.L, D.cand);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, ctx->orb_pin_a.reserve(64 * (size_t)nb + 64));
    int32_t* h_lvl = (int32_t*)ctx->orb_pin_a.p;
    SFM_CUDA(ctx, cudaMemcpyAsync(h_lvl, D.lvl, 64 * (size_t)nb, cudaMemcpyDeviceToHost, st));
    double t1 = now_ms(); tm[0] += t1 - t0;
    SFM_CUDA(ctx, cudaStreamSynchronize(st));
    double t2 = now_ms(); tm[1] += t2 - t1;
    // ---- round trip 1: candidates of every image (raster order per level)
    std::vector<int32_t> lvl(h_lvl, h_lvl + 16 * (size_t)nb);
    std::vector<size_t> cand_at(nb + 1, 0);
    for (int s = 0; s < nb; s++) {
        if (lvl[16 * s + ORB_LEVELS] > G.L[s].cand_cap) return sfmb200_fail(ctx, SFMB200_ERR_CUDA, "candidate buffer overflow (internal)");
        cand_at[s + 1] = cand_at[s] + lvl[16 * s + ORB_LEVELS];
    }
    const size_t total_cand = cand_at[nb];
    SFM_CUDA(ctx, ctx->orb_pin_b.reserve(8 * total_cand + 64));
    uint2* h_cand = (uint2*)ctx->orb_pin_b.p;
    for (int s = 0; s < nb; s++) {
        const size_t n = cand_at[s + 1] - cand_at[s];
        if (n) SFM_CUDA(ctx, cudaMemcpyAsync(h_cand + cand_at[s], D.cand + G.L[s].cand0, 8 * n, cudaMemcpyDeviceToHost, st));
    }
    SFM_CUDA(ctx, cudaStreamSynchronize(st));
    double t3 = now_ms(); tm[2] += t3 - t2;
    // ---- first selection: best 2 * quota FAST scores per (image, level); KeyPointsFilter::retainBest keeps ties
    pool.parallel_for(nb * ORB_LEVELS, [&](int t) {
        const int s = t / ORB_LEVELS, l = t % ORB_LEVELS;
        const int b = lvl[16 * s + l], e = lvl[16 * s + l + 1];
        std::vector<Rec>& r = task[t];
        r.resize(e - b);
        const uint2* c = h_cand + cand_at[s];
        for (int k = b; k < e; k++) r[k - b] = Rec{(float)(c[k].y & 0xFFFF), k};
        retain_best(r, 2 * G.L[s].lv[l].quota);
    });
    std::vector<size_t> sel_at((size_t)nb * ORB_LEVELS + 1, 0);
    for (int t = 0; t < nb * ORB_LEVELS; t++) sel_at[t + 1] = sel_at[t] + task[t].size();
    const size_t nsel = sel_at[(size_t)nb * ORB_LEVELS];
    SFM_CUDA(ctx, ctx->orb_pin_c.reserve(Carver::pad(8 * nsel + 16) * 2 + Carver::pad(4 * nsel + 16) * 2 + 1024));
    Carver pc(ctx->orb_pin_c.p);
    uint2* h_sel = pc.take<uint2>(nsel + 2); float* h_resp = pc.take<float>(nsel + 4);
    uint2* h_fin = pc.take<uint2>(nsel + 2); float* h_fresp = pc.take<float>(nsel + 4);
    pool.parallel_for(nb * ORB_LEVELS, [&](int t) {
        const int s = t / ORB_LEVELS, l = t % ORB_LEVELS;
        const uint2* c = h_cand + cand_at[s];
        uint2* o = h_sel + sel_at[t];
        for (const Rec& r : task[t]) *o++ = make_uint2(c[r.idx].x, (unsigned)l | ((unsigned)s << 8));
    });
    SFM_CUDA(ctx, ctx->orb_lists.reserve(Carver::pad(8 * nsel + 16) * 2 + Carver::pad(4 * nsel + 16) * 2 + Carver::pad(28 * nsel + 32) + Carver::pad(32 * nsel + 32) + 4096));
    Carver lc(ctx->orb_lists.p);
    uint2* d_sel = lc.take<uint2>(nsel + 2); float* d_resp = lc.take<float>(nsel + 4);
    uint2* d_fin = lc.take<uint2>(nsel + 2); float* d_fresp = lc.take<float>(nsel + 4);
    KeyPointOut* d_kp = lc.take<KeyPointOut>(nsel + 1); uint8_t* d_desc = lc.take<uint8_t>(32 * nsel + 32);
    double t4 = now_ms(); tm[3] += t4 - t3;
    if (nsel) {
        SFM_CUDA(ctx, cudaMemcpyAsync(d_sel, h_sel, 8 * nsel, cudaMemcpyHostToDevice, st));
        orb_harris_kernel<<<(unsigned)ceil_div64((int64_t)nsel * 32, 256), 256, 0, st>>>(D.pyr, D.L, d_sel, (int)nsel, d_resp);
        SFM_LAUNCH_CHECK(ctx);
        SFM_CUDA(ctx, cudaMemcpyAsync(h_resp, d_resp, 4 * nsel, cudaMemcpyDeviceToHost, st));
        SFM_CUDA(ctx, cudaStreamSynchronize(st));                                              // round trip 2
    }
    double t5 = now_ms(); tm[4] += t5 - t4;
    // ---- second selection: best quota Harris responses per (image, level)
    pool.parallel_for(nb * ORB_LEVELS, [&](int t) {
        const int s = t / ORB_LEVELS, l = t % ORB_LEVELS;
        const int n = (int)(sel_at[t + 1] - sel_at[t]);
        std::vector<Rec>& r = task[t];
        r.resize(n);
        const float* rs = h_resp + sel_at[t];
        for (int k = 0; k < n; k++) r[k] = Rec{rs[k], k};
        retain_best(r, G.L[s].lv[l].quota);
    });
    std::vector<size_t> fin_at((size_t)nb * ORB_LEVELS + 1, 0);
    for (int t = 0; t < nb * ORB_LEVELS; t++) fin_at[t + 1] = fin_at[t] + task[t].size();
    const size_t nfin = fin_at[(size_t)nb * ORB_LEVELS];
    pool.parallel_for(nb * ORB_LEVELS, [&](int t) {
        uint2* o = h_fin + fin_at[t]; float* f = h_fresp + fin_at[t];
        const uint2* src = h_sel + sel_at[t];
        for (const Rec& r : task[t]) { *o++ = src[r.idx]; *f++ = r.response; }
    });
    double t6 = now_ms(); tm[5] += t6 - t5;
    if (nfin) {
        SFM_CUDA(ctx, ctx->orb_pin_a.reserve((28 + 32) * nfin + 256));
        KeyPointOut* h_kp = (KeyPointOut*)ctx->orb_pin_a.p; uint8_t* h_desc = (uint8_t*)(h_kp + nfin);
        SFM_CUDA(ctx, cudaMemcpyAsync(d_fin, h_fin, 8 * nfin, cudaMemcpyHostToDevice, st));
        SFM_CUDA(ctx, cudaMemcpyAsync(d_fresp, h_fresp, 4 * nfin, cudaMemcpyHostToDevice, st));
        SFM_CUDA(ctx, cudaStreamWaitEvent(st, ctx->orb_ev[1], 0));
        orb_describe_kernel<<<(unsigned)ceil_div64((int64_t)nfin * 32, 256), 256, 0, st>>>(D.pyr, D.blur, D.L, d_fin, d_fresp, (int)nfin, d_kp, d_desc);
        SFM_LAUNCH_CHECK(ctx);
        SFM_CUDA(ctx, cudaMemcpyAsync(h_kp, d_kp, 28 * nfin, cudaMemcpyDeviceToHost, st));
        SFM_CUDA(ctx, cudaMemcpyAsync(h_desc, d_desc, 32 * nfin, cudaMemcpyDeviceToHost, st));
        SFM_CUDA(ctx, cudaStreamSynchronize(st));                                              // round trip 3
        double t7 = now_ms(); tm[6] += t7 - t6;
        pool.parallel_for(nb, [&](int s) {
            const size_t at = fin_at[(size_t)s * ORB_LEVELS], n_all = fin_at[(size_t)(s + 1) * ORB_LEVELS] - at;
            const size_t n = std::min<size_t>(n_all, (size_t)cap);
            if (n) {
                memcpy(kp_out + (size_t)(i0 + s) * cap, h_kp + at, 28 * n);
                memcpy(desc_out + (size_t)(i0 + s) * cap * 32, h_desc + 32 * at, 32 * n);
            }
        });
        tm[7] += now_ms() - t7;
    }
    for (int s = 0; s < nb; s++) n_out[i0 + s] = (int32_t)(fin_at[(size_t)(s + 1) * ORB_LEVELS] - fin_at[(size_t)s * ORB_LEVELS]);
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->orb_stream));        // the next group (and a download for inspection) reuses the blur buffer
    return SFMB200_OK;
}

// n_images images of sizes ws[i] x hs[i] from `in`: one plan per distinct size, groups by device bytes (orb_groups.h), and per group the
// input stage, then the shared rest.
int orb_run(sfmb200_ctx* ctx, const OrbInput& in, int n_images, const int* ws, const int* hs, int nfeatures, int cap, KeyPointOut* kp_out,
            uint8_t* desc_out, int32_t* n_out) {
    const bool host = in.host != nullptr;
    std::map<std::pair<int, int>, OrbPlan> plans;
    std::vector<const OrbPlan*> plan_of(n_images);
    std::vector<size_t> dev_bytes(n_images), stage_bytes(n_images);
    for (int i = 0; i < n_images; i++) {
        auto it = plans.find({ws[i], hs[i]});
        if (it == plans.end()) {
            it = plans.emplace(std::make_pair(ws[i], hs[i]), OrbPlan{}).first;
            make_plan(ws[i], hs[i], nfeatures, it->second);
            if (it->second.L.total_rows > 65535 * BT_H)
                return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "image too tall for one launch (%d pyramid rows)", it->second.L.total_rows);
        }
        plan_of[i] = &it->second;
        const size_t img_bytes = (size_t)ws[i] * hs[i] * (host ? in.channels : 3);
        dev_bytes[i] = orb_image_bytes(it->second.L, host && in.channels == 3 ? img_bytes : 0);
        stage_bytes[i] = host ? img_bytes : 0;
    }
    const std::vector<int> gstart = orb_groups(dev_bytes.data(), host ? stage_bytes.data() : nullptr, n_images);
    const int ngroups = (int)gstart.size() - 1;
    std::vector<OrbGroup> groups(ngroups);
    size_t dev_need = 0, tab_need = 0, stage_need = 0;
    int max_nb = 0;
    for (int g = 0; g < ngroups; g++) {
        OrbGroup& G = groups[g];
        make_group(plan_of, gstart[g], gstart[g + 1], in, G);
        OrbDev D;
        Carver a(nullptr), b(nullptr);
        dev_need = std::max(dev_need, carve(a, G, D));
        tab_need = std::max(tab_need, carve_tables(b, G, D));
        stage_need = std::max(stage_need, G.stage);
        max_nb = std::max(max_nb, G.nb);
    }
    cudaStream_t st = ctx->stream;
    if (!ctx->orb_stream) {
        SFM_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->orb_stream, cudaStreamNonBlocking));
        SFM_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->orb_up, cudaStreamNonBlocking));
        for (auto& ev : ctx->orb_ev) SFM_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    }
    double* tm = ctx->orb_ms;
    for (int i = 0; i < 8; i++) tm[i] = 0.0;
    SFM_CUDA(ctx, ctx->orb_dev.reserve(dev_need + 4096));
    SFM_CUDA(ctx, ctx->orb_pin_tab.reserve(tab_need + 256));
    if (host) SFM_CUDA(ctx, ctx->orb_pin_img.reserve(stage_need + 256));
    std::vector<std::vector<Rec>> task((size_t)max_nb * ORB_LEVELS);
    for (OrbGroup& G : groups) {
        const double t0 = now_ms();
        OrbDev D;
        Carver cv(ctx->orb_dev.p);
        carve(cv, G, D);
        for (int s = 0; s < G.nb; s++) {
            OrbLayout& L = G.L[s];
            L.src = host ? (in.channels == 3 ? D.raw + G.raw0[s] : nullptr) : in.dev[G.i0 + s];
        }
        // the tables: packed into pinned memory with the device carve's offsets, one upload
        Carver tc(ctx->orb_pin_tab.p);
        OrbDev H;
        const size_t tab_bytes = carve_tables(tc, G, H);
        memcpy(H.L, G.L.data(), sizeof(OrbLayout) * G.L.size());
        if (!G.taps.empty()) memcpy(H.taps, G.taps.data(), 4 * G.taps.size());
        memcpy(H.blur_tiles, G.blur_tiles.data(), 4 * G.blur_tiles.size());
        memcpy(H.fast_tiles, G.fast_tiles.data(), 4 * G.fast_tiles.size());
        SFM_CUDA(ctx, cudaMemcpyAsync(ctx->orb_dev.p, ctx->orb_pin_tab.p, tab_bytes, cudaMemcpyHostToDevice, st));
        SFM_CUDA(ctx, cudaMemsetAsync(D.rowcnt, 0, 4 * G.cnt, st));
        OrbLast& o = ctx->orb_last;
        o.pyr = D.pyr; o.blur = D.blur; o.score = D.score; o.nimg = 0; o.nfeatures = nfeatures;
        o.w.clear(); o.h.clear(); o.pix0.clear();
        for (const OrbLayout& L : G.L) { o.w.push_back(L.lv[0].w); o.h.push_back(L.lv[0].h); o.pix0.push_back(L.pix0); }
        if (int rc = host ? orb_input_host(ctx, G, D, in) : orb_detect(ctx, G, D, 0, G.nb, true)) return rc;
        o.nimg = G.nb;
        if (int rc = orb_finish(ctx, G, D, cap, kp_out, desc_out, n_out, task, t0)) return rc;
    }
    return SFMB200_OK;
}

}  // namespace

// The images of sfmb200_decode_jpeg_extract_orb (jpeg.cu), already on the device: packed B,G,R rows of ws[i] x hs[i] pixels at d_bgr[i].
int orb_extract_device(sfmb200_ctx* ctx, const uint8_t* const* d_bgr, const int* ws, const int* hs, int n, int nfeatures, int max_keypoints,
                       sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints) {
    OrbInput in;
    in.dev = d_bgr;
    return orb_run(ctx, in, n, ws, hs, nfeatures, max_keypoints, (KeyPointOut*)keypoints, descriptors, n_keypoints);
}

extern "C" {

int sfmb200_orb_detect_and_compute_batch(sfmb200_ctx* ctx, const uint8_t* const* images, int n_images, int width, int height, int channels,
                                         size_t row_stride, int nfeatures, int max_keypoints, sfmb200_keypoint* keypoints,
                                         uint8_t* descriptors, int32_t* n_keypoints) {
    static_assert(sizeof(sfmb200_keypoint) == 28 && sizeof(KeyPointOut) == 28, "cv::KeyPoint layout");
    if (!ctx || n_images < 0 || !n_keypoints) return SFMB200_ERR_INVALID;
    if (n_images == 0) return SFMB200_OK;
    if (!images || !keypoints || !descriptors || max_keypoints < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (channels != 1 && channels != 3) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "channels must be 1 (grey) or 3 (BGR), got %d", channels);
    if (width < 8 || height < 8 || width > 65535 || height > 65535)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image size %dx%d outside [8, 65535]", width, height);
    if ((int64_t)width * height > ((int64_t)1 << 28))          // pyramid offsets are 32-bit: 3.3 x the image must stay below 2^31 bytes
        return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "image of %dx%d pixels is too large (limit 2^28 pixels)", width, height);
    if (row_stride == 0) row_stride = (size_t)width * channels;
    if (row_stride < (size_t)width * channels) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "row_stride smaller than a row");
    if (nfeatures < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "nfeatures < 0");
    for (int i = 0; i < n_images; i++) if (!images[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d is NULL", i);
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    OrbInput in;
    in.host = images; in.channels = channels; in.row_stride = row_stride;
    const std::vector<int> ws(n_images, width), hs(n_images, height);
    return orb_run(ctx, in, n_images, ws.data(), hs.data(), nfeatures, max_keypoints, (KeyPointOut*)keypoints, descriptors, n_keypoints);
}

int sfmb200_orb_detect_and_compute(sfmb200_ctx* ctx, const uint8_t* image, int width, int height, int channels, size_t row_stride, int nfeatures,
                                   int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints) {
    const uint8_t* one[1] = {image};
    return sfmb200_orb_detect_and_compute_batch(ctx, one, 1, width, height, channels, row_stride, nfeatures, max_keypoints, keypoints, descriptors, n_keypoints);
}

int sfmb200_orb_layout(int width, int height, int nfeatures, int32_t* level_w, int32_t* level_h, float* level_scale, int32_t* level_quota) {
    if (width < 1 || height < 1 || nfeatures < 0) return SFMB200_ERR_INVALID;
    OrbLayout L; make_layout(width, height, nfeatures, L);
    for (int l = 0; l < ORB_LEVELS; l++) {
        if (level_w) level_w[l] = L.lv[l].w;
        if (level_h) level_h[l] = L.lv[l].h;
        if (level_scale) level_scale[l] = L.lv[l].scale;
        if (level_quota) level_quota[l] = L.lv[l].quota;
    }
    return SFMB200_OK;
}

int sfmb200_orb_linear_exact_taps(int src, int dst, int32_t* i0, int32_t* i1, int32_t* weight) {
    if (src < 1 || dst < 1 || !i0 || !i1 || !weight) return SFMB200_ERR_INVALID;
    linear_exact_taps(src, dst, i0, i1, weight);
    return SFMB200_OK;
}

int sfmb200_orb_retain_best(const float* response, int n, int n_points, int32_t* order) {
    if (n < 0 || (n && (!response || !order))) return -1;
    std::vector<Rec> k(n);
    for (int i = 0; i < n; i++) k[i] = Rec{response[i], i};
    retain_best(k, n_points);
    for (size_t i = 0; i < k.size(); i++) order[i] = k[i].idx;
    return (int)k.size();
}

int64_t sfmb200_host_pool_selftest(int n_threads, int rounds, int max_tasks) {
    if (n_threads < 1 || rounds < 0 || max_tasks < 0) return -1;
    HostPool pool(n_threads - 1);
    int64_t total = 0;
    for (int r = 0; r < rounds; r++) {
        const int n = max_tasks ? (r * 7919) % (max_tasks + 1) : 0;
        std::vector<int64_t> out((size_t)n, 0);
        pool.parallel_for(n, [&](int i) { int64_t a = 0; for (int k = 0; k <= i % 97; k++) a += k; out[i] = a + i; });
        for (int i = 0; i < n; i++) { int64_t a = 0; for (int k = 0; k <= i % 97; k++) a += k; if (out[i] != a + i) return -2; total += out[i]; }
    }
    return total;
}

int sfmb200_orb_last_timings(const sfmb200_ctx* ctx, double* ms8) {
    if (!ctx || !ms8) return SFMB200_ERR_INVALID;
    for (int i = 0; i < 8; i++) ms8[i] = ctx->orb_ms[i];
    return SFMB200_OK;
}

int sfmb200_orb_download_level(sfmb200_ctx* ctx, int stage, int image, int level, uint8_t* out) {
    if (!ctx || !out || level < 0 || level >= ORB_LEVELS) return SFMB200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    const OrbLast& o = ctx->orb_last;
    if (!o.pyr || image < 0 || image >= o.nimg) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "no extraction to inspect (image %d of %d)", image, o.nimg);
    OrbLayout L; make_layout(o.w[image], o.h[image], o.nfeatures, L);
    const uint8_t* base = stage == 0 ? o.pyr : stage == 1 ? o.blur : stage == 2 ? o.score : nullptr;
    if (!base) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "stage must be 0 (pyramid), 1 (blurred) or 2 (FAST score)");
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    if (L.lv[level].w == 0) return SFMB200_OK;
    SFM_CUDA(ctx, cudaMemcpyAsync(out, base + o.pix0[image] + L.lv[level].off, (size_t)L.lv[level].w * L.lv[level].h, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SFMB200_OK;
}

}  // extern "C"
