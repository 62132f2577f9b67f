// tests/host_resize.cpp -- TEST HARNESS: runs the image downscale's arithmetic (csrc/resize_math.cuh) on the CPU the way
// csrc/resize.cu does: the output size, the taps of rz_taps, and per output pixel either the 2x2 area rule (factor 0.5) or the
// horizontal pass of its two source rows followed by the vertical pass.  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/resize_math.cuh"
#include <vector>

extern "C" {

int hr_size(int w, int h, double s, int* dw, int* dh) { return rz_size(w, h, s, *dw, *dh) ? 0 : 1; }

// src: h rows of w * 3 bytes; dst: dh rows of dw * 3 bytes (sizes from hr_size).
int hr_resize(const uint8_t* src, int w, int h, double s, uint8_t* dst) {
    int dw = 0, dh = 0;
    if (!rz_size(w, h, s, dw, dh)) return 1;
    const long long stride = (long long)w * 3;
    if (rz_is_area2(s)) {
        for (int y = 0; y < dh; ++y)
            for (int x = 0; x < dw; ++x)
                for (int c = 0; c < 3; ++c) dst[((long long)y * dw + x) * 3 + c] = rz_area2(src, stride, w, h, x, y, c);
        return 0;
    }
    std::vector<RzTap> tx(dw), ty(dh);
    rz_taps(w, h, dw, dh, s, tx.data(), ty.data());
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x)
            for (int c = 0; c < 3; ++c) {
                const int32_t A0 = rz_hpass(src + ty[y].i0 * stride, tx[x], c), A1 = rz_hpass(src + ty[y].i1 * stride, tx[x], c);
                dst[((long long)y * dw + x) * 3 + c] = rz_vpass(A0, A1, ty[y].a0, ty[y].a1);
            }
    return 0;
}

}  // extern "C"
