// resize_math.cuh -- the arithmetic of the image downscale (csrc/resize.cu), __host__ __device__ so that the CPU tests compile it with g++.
//
// What cv::resize(src, dst, Size(), s, s) returns for an 8-bit B,G,R image with the default INTER_LINEAR in OpenCV 4.13:
//   - output size dw = cvRound(w * s), dh = cvRound(h * s) (half to even); the map scale is 1.0 / s, not w / dw;
//   - an output of the input's size is a copy of it (cv::resize's dsize == ssize shortcut);
//   - 1.0 / s == 2 exactly: the fast INTER_AREA path, (a + b + c + d + 2) >> 2 of each 2x2 block, where a block cut by the right or
//     bottom edge (odd sizes that round up) averages its in-bounds pixels, cvRound((float)sum / count);
//   - any other factor: fixed-point bilinear with Q11 weights.  Column taps are clamped to [0, w - 1] with weight (2048, 0) at either
//     end; row taps clamp only their indices, so the first and last rows mix a row with itself.  Horizontal pass in int32; vertical
//     pass with the rounding of OpenCV's SIMD kernel (VResizeLinearVec_32s8u), which it applies to every pixel.
// The taps are computed on the host (rz_tap): their float / double arithmetic decides the weights, so it is kept apart from any
// fused multiply-add.  Identity taps (i, i, 2048, 0) reproduce the input exactly, so a same-size image needs no separate path.
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define RZ_HD __host__ __device__
#else
#define RZ_HD
#endif
#define RZ_FI RZ_HD inline

constexpr int RZ_COEF_ONE = 2048;       // INTER_RESIZE_COEF_SCALE (Q11)

// One output column or row: its two source indices and their Q11 weights.
struct RzTap { int32_t i0, i1, a0, a1; };

// One image of a batch: source and destination offsets in one device buffer each, rows of src_stride / dst_stride bytes, its first
// column tap and first row tap in the batch's tap table, and its output tiles (tiles_x per tile row, ntiles in all).
struct RzImg {
    int sw, sh, dw, dh;
    long long src0, dst0, src_stride, dst_stride;
    int tap_x, tap_y, tiles_x, ntiles;
};

// cvRound of a double: round half to even (the default rounding mode).
inline long long rz_round(double v) { return std::llrint(v); }

// Output size of cv::resize for factor s; false where cv::resize asserts (s not finite or <= 0, empty or oversized output).
inline bool rz_size(int w, int h, double s, int& dw, int& dh) {
    if (!std::isfinite(s) || s <= 0 || w <= 0 || h <= 0) return false;
    const double fw = (double)w * s, fh = (double)h * s;
    if (!(fw < 2147483647.0 && fh < 2147483647.0)) return false;
    const long long rw = rz_round(fw), rh = rz_round(fh);
    if (rw < 1 || rh < 1) return false;
    dw = (int)rw; dh = (int)rh;
    return true;
}

// cv::resize takes its fast 2x2 area path when both map scales are exactly 2.
inline bool rz_is_area2(double s) { return 1.0 / s == 2.0; }

// Tap of output column (clamp_weights) or row d of a map from n source pixels at map scale inv = 1.0 / s (resizeGeneric_'s
// coefficient loops).  Host only.
inline RzTap rz_tap(int d, double inv, int n, bool clamp_weights) {
    volatile double p = ((double)d + 0.5) * inv;     // kept a separate rounding: a fused multiply-add would move some weights
    float f = (float)(p - 0.5);
    int i = (int)std::floor(f);
    f -= (float)i;
    RzTap t;
    if (clamp_weights) {
        if (i < 0) { i = 0; f = 0.f; }
        if (i >= n - 1) { i = n - 1; f = 0.f; }
        t.i0 = i; t.i1 = i + 1 < n ? i + 1 : n - 1;
    } else {
        t.i0 = i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
        t.i1 = i + 1 < 0 ? 0 : (i + 1 > n - 1 ? n - 1 : i + 1);
    }
    t.a0 = (int32_t)std::lrint((1.f - f) * (float)RZ_COEF_ONE);
    t.a1 = (int32_t)std::lrint(f * (float)RZ_COEF_ONE);
    return t;
}

// The dw column taps tx and dh row taps ty of a sw x sh image resized to dw x dh by factor s.  Host only.
inline void rz_taps(int sw, int sh, int dw, int dh, double s, RzTap* tx, RzTap* ty) {
    const bool copy = dw == sw && dh == sh;          // cv::resize copies an image whose size does not change: identity taps
    const double inv = 1.0 / s;
    for (int x = 0; x < dw; ++x) tx[x] = copy ? RzTap{x, x, RZ_COEF_ONE, 0} : rz_tap(x, inv, sw, true);
    for (int y = 0; y < dh; ++y) ty[y] = copy ? RzTap{y, y, RZ_COEF_ONE, 0} : rz_tap(y, inv, sh, false);
}

// Horizontal pass of channel c of one B,G,R source row.
RZ_FI int32_t rz_hpass(const uint8_t* row, const RzTap& t, int c) {
    return (int32_t)row[3 * t.i0 + c] * t.a0 + (int32_t)row[3 * t.i1 + c] * t.a1;
}

// Vertical pass: OpenCV's SIMD rounding, (A >> 4) packed to int16, multiply-high by the Q11 weight, then (sum + 2) >> 2 saturated.
RZ_FI uint8_t rz_vpass(int32_t A0, int32_t A1, int32_t b0, int32_t b1) {
    const int32_t v = ((((A0 >> 4) * b0) >> 16) + (((A1 >> 4) * b1) >> 16) + 2) >> 2;
    return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Channel c of output pixel (dx, dy) of the 2x2 area path over a sw x sh B,G,R source with rows of `stride` bytes.
RZ_FI uint8_t rz_area2(const uint8_t* src, long long stride, int sw, int sh, int dx, int dy, int c) {
    const int x = 2 * dx, y = 2 * dy;
    const uint8_t* r0 = src + (long long)y * stride + 3 * x + c;
    if (x + 1 < sw && y + 1 < sh) return (uint8_t)((r0[0] + r0[3] + r0[stride] + r0[stride + 3] + 2) >> 2);
    const bool xr = x + 1 < sw, yr = y + 1 < sh;              // a block cut by the right or bottom edge
    const int sum = r0[0] + (xr ? r0[3] : 0) + (yr ? r0[stride] : 0);
    const int cnt = 1 + xr + yr;
    const float m = (float)sum / (float)cnt;                   // count is 1 or 2: exact, so rint is cvRound's half-to-even
#ifdef __CUDA_ARCH__
    const int v = __float2int_rn(m);
#else
    const int v = (int)std::lrint(m);
#endif
    return (uint8_t)(v > 255 ? 255 : v);
}
