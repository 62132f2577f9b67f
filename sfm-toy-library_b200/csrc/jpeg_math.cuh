// jpeg_math.cuh -- the arithmetic of the JPEG decoder (csrc/jpeg.cu), __host__ __device__ so that the CPU tests compile it with g++.
//
// What cv::imread(IMREAD_COLOR) returns with the libjpeg-turbo 3.1 that OpenCV 4.13 bundles:
//   - Huffman decoding of one codeword (symbol + appended bits) and the decoder state a codeword leaves behind (jdhuff.c);
//   - the self-synchronising span decoder of Weissenberger & Schmidt (ICPP 2018, HiPC 2021) built on it;
//   - jpeg_idct_islow (jidctint.c: LL&M, CONST_BITS 13, PASS1_BITS 2, the 10-bit wrap of the range-limit table);
//   - fancy upsampling (jdsample.c: h2v1 / h2v2 with their alternating biases, h1v2, box for h4v1 and for widths <= 2);
//   - YCbCr -> RGB with the integer tables of jdcolor.c;
//   - the EXIF orientation remap of cv::imread (flip / transpose).
// Arithmetic is done in the integer widths libjpeg uses (JLONG = 64 bit), so no input can overflow a signed type.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define JM_HD __host__ __device__
#else
#define JM_HD
#endif
#define JM_FI JM_HD inline

constexpr int JM_FAST_BITS = 9;
constexpr int JM_MAX_BPM = 10;          // blocks per MCU (the JPEG limit)

// Derived decoding table of one Huffman table (jpeg_make_d_derived_tbl): a 9-bit lookup for the short codes and the canonical
// maxcode / valoffset walk for the longer ones.
struct JmHuff {
    uint16_t fast[1 << JM_FAST_BITS];   // (length << 8) | symbol for codes of <= 9 bits, 0 otherwise
    int32_t maxcode[18];                // largest code of each length, -1 = none; [17] is a sentinel
    int32_t valoff[18];                 // symbol index of a code of length l = code + valoff[l]
    uint8_t vals[256];
};

// MCU structure of a scan: which component, and which block of its footprint, each block of an MCU is.
struct JmScan {
    int bpm;
    uint8_t blk_comp[JM_MAX_BPM], blk_dx[JM_MAX_BPM], blk_dy[JM_MAX_BPM];
    int16_t dc_tab[JM_MAX_BPM], ac_tab[JM_MAX_BPM];   // table indices per block of the MCU
};

// natural (row-major) position of zig-zag index k
JM_HD constexpr uint8_t jm_natural(int k) {
    constexpr uint8_t t[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                               28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
                               54, 47, 55, 62, 63};
    return t[k];
}

// Builds the derived table from the DHT counts (bits[1..16]) and symbols; false for a table libjpeg rejects (JERR_BAD_HUFF_TABLE).
inline bool jm_build_huff(const uint8_t* bits /*[17], bits[0] unused*/, const uint8_t* vals, int nvals, bool is_dc, JmHuff& h) {
    for (int i = 0; i < (1 << JM_FAST_BITS); ++i) h.fast[i] = 0;
    for (int i = 0; i < 256; ++i) h.vals[i] = i < nvals ? vals[i] : 0;
    int count = 0;
    for (int l = 1; l <= 16; ++l) count += bits[l];
    if (count > 256 || count != nvals) return false;
    uint32_t code = 0;
    int k = 0;
    for (int l = 1; l <= 16; ++l) {
        if (bits[l]) {
            h.valoff[l] = k - (int32_t)code;
            for (int i = 0; i < bits[l]; ++i, ++k, ++code) {
                if (l <= JM_FAST_BITS) {
                    const int shift = JM_FAST_BITS - l;
                    for (uint32_t f = code << shift; f < ((code + 1) << shift); ++f) h.fast[f] = (uint16_t)((l << 8) | vals[k]);
                }
            }
            h.maxcode[l] = (int32_t)code - 1;
        } else {
            h.valoff[l] = 0;
            h.maxcode[l] = -1;
        }
        if (code >= (1u << l)) return false;      // code space overflow or an all-ones code (libjpeg: code >= 1 << si)
        code <<= 1;
    }
    h.maxcode[0] = -1; h.valoff[0] = 0;
    h.maxcode[17] = 0x7fffffff; h.valoff[17] = 0;
    if (is_dc)
        for (int i = 0; i < nvals; ++i)
            if (vals[i] > 15) return false;
    return true;
}

// The 32 bits that start at bit p of an MSB-first stream; the buffer is padded so that 8 bytes past any valid position are readable.
JM_FI uint32_t jm_peek32(const uint8_t* buf, uint32_t p) {
#ifdef __CUDA_ARCH__
    const uint32_t* w = reinterpret_cast<const uint32_t*>(buf) + (p >> 5);      // buf is 4-byte aligned on the device
    const uint32_t a = __byte_perm(__ldg(w), 0, 0x0123), b = __byte_perm(__ldg(w + 1), 0, 0x0123);
    return __funnelshift_l(b, a, p & 31);
#else
    const uint8_t* q = buf + (p >> 3);
    const uint64_t v = ((uint64_t)q[0] << 32) | ((uint64_t)q[1] << 24) | ((uint64_t)q[2] << 16) | ((uint64_t)q[3] << 8) | (uint64_t)q[4];
    return (uint32_t)(v >> (8 - (p & 7)));
#endif
}

// Huffman symbol of the 16 bits at the head of `bits16`: returns its length (0 = no code of this table starts here)
JM_FI int jm_huff(const JmHuff& h, uint32_t bits16, int& sym) {
    const uint16_t f = h.fast[bits16 >> (16 - JM_FAST_BITS)];
    if (f) { sym = f & 0xff; return f >> 8; }
    for (int l = JM_FAST_BITS + 1; l <= 16; ++l) {
        const int32_t code = (int32_t)(bits16 >> (16 - l));
        if (code <= h.maxcode[l]) { sym = h.vals[(code + h.valoff[l]) & 0xff]; return l; }
    }
    return 0;
}

// One codeword at bit p: the Huffman symbol and its appended bits, read within [p, end).  zz is the zig-zag index the codeword
// belongs to (0 = DC); on return it is the next one, 64 when the block is complete.  *k = zig-zag index written (-1 = none), *v the
// value (the DC difference for k = 0).  Returns false where no codeword of the table starts, the codeword overruns `end`, or an AC
// run leaves the block (libjpeg would write past coefficient 63); p is left unchanged then.
JM_FI bool jm_step(const uint8_t* buf, uint32_t& p, uint32_t end, const JmHuff& h, int& zz, int& k, int& v) {
    if (p >= end) return false;
    const uint32_t bits = jm_peek32(buf, p);
    int sym = 0;
    const int len = jm_huff(h, bits >> 16, sym);
    if (!len) return false;
    const int s = sym & 15, r = sym >> 4;
    const uint32_t total = (uint32_t)(len + s);
    if (total > end - p) return false;
    int val = 0;
    if (s) {
        const int x = (int)((bits << len) >> (32 - s));
        val = x < (1 << (s - 1)) ? x - (1 << s) + 1 : x;                        // HUFF_EXTEND
    }
    if (zz == 0) { k = 0; v = val; zz = 1; }
    else if (s) {
        const int kk = zz + r;
        if (kk > 63) return false;
        k = kk; v = val; zz = kk + 1;
    } else if (r == 15) { k = -1; v = 0; zz = zz + 16 > 64 ? 64 : zz + 16; }       // ZRL (a run past 63 ends the block, as in libjpeg)
    else { k = -1; v = 0; zz = 64; }                                               // EOB
    p += total;
    return true;
}

// ------------------------------------------------------------------------------------------------ self-synchronising decoding
// A segment (the entropy-coded data between restart markers) is cut into subsequences of S bits.  The decoder state at a codeword
// boundary is (block of the MCU, zig-zag index); jm_span decodes from an entry (bit position, state) until the first codeword
// boundary at or past `stop` and returns that exit, packed with the number of blocks begun on the way.  Where no codeword starts
// (a wrong guess of the state, or the end of the data) it moves on one bit at a block start, so a span always ends.
// The exits of a segment are a fixed point: exit[j] = span(exit[j-1]) with exit[-1] = (segment start, 0).  Starting every
// subsequence from a guessed state and re-decoding a subsequence whenever its predecessor's exit changed reaches it.  A wrong
// guess of the block within the MCU can decode plausibly for a while, so it takes a few rounds (csrc/jpeg.cu).
JM_FI uint64_t jm_pack_exit(uint32_t pos, int state, int nblk) { return ((uint64_t)pos << 32) | ((uint64_t)(uint32_t)nblk << 10) | (uint32_t)state; }
JM_FI uint32_t jm_exit_pos(uint64_t e) { return (uint32_t)(e >> 32); }
JM_FI int jm_exit_state(uint64_t e) { return (int)(e & 1023); }
JM_FI int jm_exit_nblk(uint64_t e) { return (int)((uint32_t)e >> 10); }
// two exits continue identically iff position and state agree (the block count only places the blocks decoded before them)
JM_FI bool jm_exit_same(uint64_t a, uint64_t b) { return (a >> 32) == (b >> 32) && (a & 1023) == (b & 1023); }

struct JmNoSink {
    JM_FI void coef(int, int, int) {}
    JM_FI void fail(int, int) {}
};

// Decodes from (p, state) until a codeword boundary >= stop; reads never pass seg_end.  The sink sees every coefficient as
// (block ordinal counted from the entry, zig-zag index, value) -- the ordinal is -1 for a block begun before the entry -- and every
// position where no codeword starts as fail(ordinal of the block being decoded, zig-zag index).  `ncw` counts codewords.
template <class Sink>
JM_FI uint64_t jm_span(const uint8_t* buf, uint32_t p, int state, uint32_t stop, uint32_t seg_end, const JmScan& sc, const JmHuff* tabs,
                       Sink& sink, int* ncw = nullptr) {
    int blk = state >> 6, zz = state & 63, nblk = 0, cw = 0;
    while (p < stop) {
        const JmHuff& h = tabs[zz == 0 ? sc.dc_tab[blk] : sc.ac_tab[blk]];
        int k = -1, v = 0;
        if (!jm_step(buf, p, seg_end, h, zz, k, v)) {
            sink.fail(nblk - 1 + (zz == 0), zz);
            p += 1; blk = 0; zz = 0;
            continue;
        }
        ++cw;
        if (k == 0) ++nblk;
        if (k >= 0) sink.coef(nblk - 1, k, v);
        if (zz == 64) { zz = 0; if (++blk == sc.bpm) blk = 0; }
    }
    if (ncw) *ncw += cw;
    return jm_pack_exit(p, blk * 64 + zz, nblk);
}

// ------------------------------------------------------------------------------------------------ jpeg_idct_islow
// coef [64] natural order, quant [64] natural order (ISLOW_MULT_TYPE is short in a SIMD build); out rows of 8 bytes, stride ostride
JM_FI uint8_t jm_range_limit(long long x) {          // sample_range_limit[CENTERJSAMPLE + (x & RANGE_MASK)]
    const int t = (int)(x & 1023);
    const int s = t >= 512 ? t - 1024 : t;
    const int o = s + 128;
    return (uint8_t)(o < 0 ? 0 : (o > 255 ? 255 : o));
}

// The odd/even butterflies of one 8-point pass; in[i] already dequantised (pass 1) or the work array (pass 2).
JM_FI void jm_idct_1d(const long long* in, long long* out, int shift, long long round_add) {
    typedef long long J;
    const J F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
            F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    J z2 = in[2], z3 = in[6];
    J z1 = (z2 + z3) * F0541;
    J tmp2 = z1 + z3 * (-F1847);
    J tmp3 = z1 + z2 * F0765;
    z2 = in[0]; z3 = in[4];
    J tmp0 = (J)((unsigned long long)(z2 + z3) << 13);
    J tmp1 = (J)((unsigned long long)(z2 - z3) << 13);
    const J tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = in[7]; tmp1 = in[5]; tmp2 = in[3]; tmp3 = in[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    J z4 = tmp1 + tmp3;
    const J z5 = (z3 + z4) * F1175;
    tmp0 = tmp0 * F0298; tmp1 = tmp1 * F2053; tmp2 = tmp2 * F3072; tmp3 = tmp3 * F1501;
    z1 = z1 * (-F0899); z2 = z2 * (-F2562); z3 = z3 * (-F1961); z4 = z4 * (-F0390);
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    out[0] = (tmp10 + tmp3 + round_add) >> shift;
    out[7] = (tmp10 - tmp3 + round_add) >> shift;
    out[1] = (tmp11 + tmp2 + round_add) >> shift;
    out[6] = (tmp11 - tmp2 + round_add) >> shift;
    out[2] = (tmp12 + tmp1 + round_add) >> shift;
    out[5] = (tmp12 - tmp1 + round_add) >> shift;
    out[3] = (tmp13 + tmp0 + round_add) >> shift;
    out[4] = (tmp13 - tmp0 + round_add) >> shift;
}

// pass 1 on column c: dequantise and transform, result (int, like libjpeg's workspace) into ws[c + 8 r]
JM_FI void jm_idct_col(const int16_t* coef, const int16_t* quant, int c, int* ws) {
    long long in[8], out[8];
    bool ac_zero = true;
    for (int r = 0; r < 8; ++r) {
        in[r] = (long long)((int)coef[8 * r + c] * (int)quant[8 * r + c]);
        if (r && coef[8 * r + c]) ac_zero = false;
    }
    if (ac_zero) {                                   // the DC-only shortcut keeps libjpeg's int arithmetic
        const int dc = (int)((unsigned)(int)in[0] << 2);
        for (int r = 0; r < 8; ++r) ws[8 * r + c] = dc;
        return;
    }
    jm_idct_1d(in, out, 11, 1ll << 10);              // DESCALE(x, CONST_BITS - PASS1_BITS)
    for (int r = 0; r < 8; ++r) ws[8 * r + c] = (int)out[r];
}

// pass 2 on row r of the workspace -> 8 samples
JM_FI void jm_idct_row(const int* ws, int r, uint8_t* o) {
    long long in[8], out[8];
    for (int c = 0; c < 8; ++c) in[c] = ws[8 * r + c];
    jm_idct_1d(in, out, 18, 1ll << 17);              // DESCALE(x, CONST_BITS + PASS1_BITS + 3)
    for (int c = 0; c < 8; ++c) o[c] = jm_range_limit(out[c]);
}

// ------------------------------------------------------------------------------------------------ upsampling and colour
// One upsampled chroma sample at full-resolution (x, y) from a plane of cw x ch samples (row stride `stride`), for the ratios
// hr = max_h / h and vr = max_v / v of the component.  libjpeg-turbo's choice (jinit_upsampler): h2v1 and h2v2 are fancy when the
// component is more than 2 samples wide, h1v2 is always fancy, everything else is pixel replication.
JM_FI int jm_chroma(const uint8_t* pl, int stride, int cw, int ch, int hr, int vr, int x, int y) {
    if (hr == 1 && vr == 1) return pl[(long long)y * stride + x];
    if (hr == 2 && vr == 1 && cw > 2) {
        const uint8_t* row = pl + (long long)y * stride;
        const int i = x >> 1;
        if ((x & 1) == 0) return (row[i] * 3 + row[i > 0 ? i - 1 : 0] + 1) >> 2;
        return (row[i] * 3 + row[i + 1 < cw ? i + 1 : cw - 1] + 2) >> 2;
    }
    if (hr == 1 && vr == 2) {
        const int r = y >> 1;
        const int f = (y & 1) ? (r + 1 < ch ? r + 1 : ch - 1) : (r > 0 ? r - 1 : 0);
        return (pl[(long long)r * stride + x] * 3 + pl[(long long)f * stride + x] + ((y & 1) ? 2 : 1)) >> 2;
    }
    if (hr == 2 && vr == 2 && cw > 2) {
        const int r = y >> 1, i = x >> 1;
        const int f = (y & 1) ? (r + 1 < ch ? r + 1 : ch - 1) : (r > 0 ? r - 1 : 0);
        const uint8_t* n = pl + (long long)r * stride;
        const uint8_t* fr = pl + (long long)f * stride;
        const int j = (x & 1) ? (i + 1 < cw ? i + 1 : cw - 1) : (i > 0 ? i - 1 : 0);
        const int cs = n[i] * 3 + fr[i], os = n[j] * 3 + fr[j];
        return (x & 1) ? (cs * 3 + os + 7) >> 4 : (cs * 3 + os + 8) >> 4;
    }
    return pl[(long long)(y / vr) * stride + x / hr];
}

// ycc_rgb_convert with the tables of build_ycc_rgb_table (SCALEBITS 16); writes B, G, R
JM_FI void jm_ycc_to_bgr(int y, int cb, int cr, uint8_t* bgr) {
    const long long x_cb = cb - 128, x_cr = cr - 128;
    const int r = y + (int)((91881ll * x_cr + 32768) >> 16);
    const int g = y + (int)(((-22554ll * x_cb + 32768) + (-46802ll * x_cr)) >> 16);
    const int b = y + (int)((116130ll * x_cb + 32768) >> 16);
    bgr[0] = (uint8_t)(b < 0 ? 0 : (b > 255 ? 255 : b));
    bgr[1] = (uint8_t)(g < 0 ? 0 : (g > 255 ? 255 : g));
    bgr[2] = (uint8_t)(r < 0 ? 0 : (r > 255 ? 255 : r));
}

// Source pixel (x, y) of output pixel (ox, oy) of an image of W x H decoded pixels under EXIF orientation o (cv::imread's flips and
// transposes); a transposing orientation (5-8) gives an H x W output.
JM_FI void jm_orient_src(int o, int W, int H, int ox, int oy, int& x, int& y) {
    switch (o) {
    case 2: x = W - 1 - ox; y = oy; break;
    case 3: x = W - 1 - ox; y = H - 1 - oy; break;
    case 4: x = ox; y = H - 1 - oy; break;
    case 5: x = oy; y = ox; break;
    case 6: x = oy; y = H - 1 - ox; break;
    case 7: x = W - 1 - oy; y = H - 1 - ox; break;
    case 8: x = W - 1 - oy; y = ox; break;
    default: x = ox; y = oy; break;
    }
}
