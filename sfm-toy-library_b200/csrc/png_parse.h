// png_parse.h -- host side of the PNG decoder (csrc/png.cu): the chunk walk with CRC-32, IHDR, PLTE, the EXIF orientation of an eXIf
// chunk, the zlib header and the raw (filtered) size of every Adam7 pass.  Plain C++ (no CUDA), so that the CPU tests compile it with
// g++ and the sanitizers.  No inflate runs here: the IDAT payloads go to the device as they are.
//
// The rules are libpng 1.6's as cv::imread(IMREAD_COLOR) meets them: a CRC error in a critical chunk (IHDR, PLTE, IDAT, IEND) fails,
// one in an ancillary chunk drops that chunk; every ancillary chunk but eXIf is ignored (tRNS, gAMA, sRGB, iCCP, sBIT, cHRM: alpha
// and colour management do not reach an IMREAD_COLOR image); bytes after IEND are ignored.  APNG files (acTL) are refused as
// unsupported rather than decoded to their default image.
#pragma once
#include "jpeg_parse.h"
#include "png_math.cuh"
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

struct PgImage {
    int W = 0, H = 0, bd = 0, ct = 0, interlace = 0, orient = 1, OW = 0, OH = 0;
    int channels = 0, bpp = 0;                    // samples per pixel; bytes per complete pixel for the filters (at least 1)
    int npal = 0;
    uint8_t pal[256 * 3] = {};                    // R,G,B, zero past npal
    int64_t pw[7] = {}, ph[7] = {}, prow[7] = {}, poff[7] = {};   // pass size in pixels, row bytes (filter byte excluded), raw offset
    int npass = 1;
    int64_t raw = 0;                              // filtered bytes of all passes
    std::vector<std::pair<size_t, size_t>> idat;  // (offset, length) of every IDAT payload
    size_t zlen = 0;                              // IDAT bytes in all
};

inline uint32_t pg_crc32(const uint8_t* p, size_t n) {
    static uint32_t tab[256];
    static bool init = [] {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            tab[i] = c;
        }
        return true;
    }();
    (void)init;
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

inline bool pg_is_png(const uint8_t* d, size_t n) {
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    return d && n >= 8 && !memcmp(d, sig, 8);
}

inline uint32_t pg_be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

// Row bytes of `w` pixels (filter byte excluded)
inline int64_t pg_rowbytes(int64_t w, int channels, int bd) { return (w * channels * bd + 7) / 8; }

// Parses the file.  Returns JP_OK / JP_INVALID / JP_UNSUPPORTED (the SFMB200 codes) with the reason in `why`.  max_raw: the largest
// raw size the device indexing takes.
inline int pg_parse(const uint8_t* data, size_t size, PgImage& im, std::string& why, int64_t max_raw = ((int64_t)1 << 31) - 1) {
    auto fail = [&](int code, const char* fmt, ...) {
        char buf[256];
        va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
        why = buf;
        return code;
    };
    if (!pg_is_png(data, size)) return fail(JP_INVALID, "not a PNG file (no PNG signature)");
    size_t i = 8;
    bool have_ihdr = false, have_plte = false, have_exif = false, in_idat = false, idat_done = false;
    for (;;) {
        if (size - i < 12) return fail(JP_INVALID, "file ends inside a chunk at byte %zu (truncated or no IEND)", i);
        const uint32_t len = pg_be32(data + i);
        const uint8_t* type = data + i + 4;
        if (len > 0x7FFFFFFFu || size - i - 12 < len) return fail(JP_INVALID, "chunk at byte %zu: length %u past the end of the file", i, len);
        char name[5] = {0, 0, 0, 0, 0};
        for (int k = 0; k < 4; ++k) {
            const uint8_t c = type[k];
            if (!((c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'))) return fail(JP_INVALID, "chunk at byte %zu: invalid chunk type", i);
            name[k] = (char)c;
        }
        const uint8_t* p = type + 4;
        const bool critical = !(type[0] & 0x20);
        const bool crc_ok = pg_crc32(type, len + 4) == pg_be32(p + len);
        const size_t at = i;
        i += 12 + (size_t)len;
        if (!crc_ok) {
            if (critical) return fail(JP_INVALID, "%s chunk at byte %zu: CRC error", name, at);
            continue;                                        // an ancillary chunk with a bad CRC is dropped
        }
        const bool is_idat = !memcmp(type, "IDAT", 4);
        if (!have_ihdr && memcmp(type, "IHDR", 4)) return fail(JP_INVALID, "%s chunk before IHDR", name);
        if (in_idat && !is_idat) { in_idat = false; idat_done = true; }
        if (!memcmp(type, "IHDR", 4)) {
            if (have_ihdr) return fail(JP_INVALID, "two IHDR chunks");
            if (len != 13) return fail(JP_INVALID, "IHDR of %u bytes", len);
            have_ihdr = true;
            const uint32_t W = pg_be32(p), H = pg_be32(p + 4);
            im.bd = p[8]; im.ct = p[9]; im.interlace = p[12];
            if (W == 0 || H == 0 || W > 0x7FFFFFFFu || H > 0x7FFFFFFFu) return fail(JP_INVALID, "image size %ux%u", W, H);
            if (W > 1000000u || H > 1000000u) return fail(JP_INVALID, "image size %ux%u exceeds libpng's limit of 1000000 per side", W, H);
            const int bd = im.bd, ct = im.ct;
            bool ok = false;
            switch (ct) {
            case 0: ok = bd == 1 || bd == 2 || bd == 4 || bd == 8 || bd == 16; im.channels = 1; break;
            case 2: ok = bd == 8 || bd == 16; im.channels = 3; break;
            case 3: ok = bd == 1 || bd == 2 || bd == 4 || bd == 8; im.channels = 1; break;
            case 4: ok = bd == 8 || bd == 16; im.channels = 2; break;
            case 6: ok = bd == 8 || bd == 16; im.channels = 4; break;
            default: break;
            }
            if (!ok) return fail(JP_INVALID, "colour type %d with bit depth %d", ct, bd);
            if (p[10] != 0 || p[11] != 0 || im.interlace > 1) return fail(JP_INVALID, "compression %d / filter %d / interlace %d method", p[10], p[11], im.interlace);
            im.W = (int)W; im.H = (int)H;
            if ((int64_t)W * H > ((int64_t)1 << 30)) return fail(JP_INVALID, "image size %ux%u exceeds cv::imread's limit of 2^30 pixels", W, H);
            im.bpp = std::max(1, im.channels * bd / 8);
        } else if (!memcmp(type, "PLTE", 4)) {
            if (have_plte) return fail(JP_INVALID, "two PLTE chunks");
            if (idat_done || in_idat) return fail(JP_INVALID, "PLTE after IDAT");
            have_plte = true;
            if (im.ct == 3) {
                if (len % 3 || len == 0 || len > 768) return fail(JP_INVALID, "PLTE of %u bytes", len);
                im.npal = (int)len / 3;
                if (im.npal > (1 << im.bd)) im.npal = 1 << im.bd;   // libpng keeps at most 2^depth entries
                memcpy(im.pal, p, 3 * (size_t)im.npal);
            }
        } else if (is_idat) {
            if (idat_done) return fail(JP_INVALID, "IDAT chunks are not consecutive");
            if (im.ct == 3 && !have_plte) return fail(JP_INVALID, "palette image without PLTE before IDAT");
            in_idat = true;
            im.idat.push_back({(size_t)(p - data), (size_t)len});
            im.zlen += len;
        } else if (!memcmp(type, "IEND", 4)) {
            break;
        } else if (!memcmp(type, "eXIf", 4)) {
            // libpng keeps the first eXIf chunk whose byte order mark is II or MM; cv::imread reads IFD0's orientation from it
            if (!have_exif && len >= 2 && p[0] == p[1] && (p[0] == 'I' || p[0] == 'M')) { have_exif = true; im.orient = jp_tiff_orientation(p, len); }
        } else if (!memcmp(type, "acTL", 4)) {
            return fail(JP_UNSUPPORTED, "animated PNG (acTL chunk)");
        } else if (critical) {
            return fail(JP_INVALID, "unknown critical chunk %s", name);
        }
    }
    if (im.idat.empty() || im.zlen == 0) return fail(JP_INVALID, "no image data (no IDAT)");
    // the zlib header: CM 8, CINFO <= 7, FCHECK, no preset dictionary
    auto zbyte = [&](size_t k) -> int {
        for (auto& c : im.idat) { if (k < c.second) return data[c.first + k]; k -= c.second; }
        return -1;
    };
    const int cmf = zbyte(0), flg = zbyte(1);
    if (cmf < 0 || flg < 0) return fail(JP_INVALID, "IDAT data shorter than a zlib header");
    if ((cmf & 15) != 8 || (cmf >> 4) > 7) return fail(JP_INVALID, "zlib header: compression method %d, window %d", cmf & 15, cmf >> 4);
    if ((cmf * 256 + flg) % 31) return fail(JP_INVALID, "zlib header: bad FCHECK");
    if (flg & 0x20) return fail(JP_INVALID, "zlib header: preset dictionary");
    // raw size of every pass
    im.npass = im.interlace ? 7 : 1;
    int64_t off = 0;
    for (int ps = 0; ps < im.npass; ++ps) {
        const int x0 = im.interlace ? pm_a7_x0(ps) : 0, y0 = im.interlace ? pm_a7_y0(ps) : 0;
        const int dx = im.interlace ? pm_a7_dx(ps) : 1, dy = im.interlace ? pm_a7_dy(ps) : 1;
        im.pw[ps] = im.W > x0 ? (im.W - x0 + dx - 1) / dx : 0;
        im.ph[ps] = im.H > y0 ? (im.H - y0 + dy - 1) / dy : 0;
        if (im.pw[ps] == 0 || im.ph[ps] == 0) im.pw[ps] = im.ph[ps] = 0;
        im.prow[ps] = pg_rowbytes(im.pw[ps], im.channels, im.bd);
        im.poff[ps] = off;
        off += im.ph[ps] * (1 + im.prow[ps]);
    }
    im.raw = off;
    if (im.raw > max_raw) return fail(JP_UNSUPPORTED, "%lld bytes of filtered image data (limit %lld)", (long long)im.raw, (long long)max_raw);
    const bool tr = im.orient >= 5;
    im.OW = tr ? im.H : im.W; im.OH = tr ? im.W : im.H;
    return JP_OK;
}
