// jpeg_parse.h -- host side of the JPEG decoder (csrc/jpeg.cu): markers, quantisation and Huffman tables, MCU layout, EXIF orientation
// and the walk over the entropy-coded data that finds the scan's end and its restart segments.  Plain C++ (no CUDA), so that the CPU
// tests compile it with g++ and the sanitizers.
//
// Supported: SOF0 / SOF1, 8-bit, 1 component or 3 components in one interleaved scan, luma sampling 1x1, 2x1, 2x2, 1x2 or 4x1 with
// 1x1 chroma (what cv::imencode writes), restart intervals, any APPn / COM.  Everything else is JP_UNSUPPORTED; data libjpeg would
// only warn about (a truncated scan, a missing or out-of-order restart marker) is JP_INVALID.
#pragma once
#include "jpeg_math.cuh"
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

enum { JP_OK = 0, JP_INVALID = 1, JP_UNSUPPORTED = 5 };   // the SFMB200_OK / _ERR_INVALID / _ERR_UNSUPPORTED codes

struct JpImage {
    int W = 0, H = 0, ncomp = 0, orient = 1, OW = 0, OH = 0;
    int hs[3] = {1, 1, 1}, vs[3] = {1, 1, 1}, hmax = 1, vmax = 1;
    int cw[3] = {0, 0, 0}, ch[3] = {0, 0, 0};     // component size in samples (downsampled_width / _height)
    int wb[3] = {0, 0, 0}, hb[3] = {0, 0, 0};     // component block grid, padded to whole MCUs
    int mcus_x = 0, mcus_y = 0, restart = 0;      // restart interval in MCUs, 0 = none
    int16_t qt[3][64];                            // per component, natural order
    JmHuff tabs[8] = {};                          // DC tables 0-3, AC tables 4-7
    JmScan scan = {};                             // table indices local to tabs
    size_t scan_off = 0, scan_len = 0;            // the entropy-coded bytes, restart markers included
    std::vector<uint32_t> seg_bytes;              // bytes of every restart segment after unstuffing
    std::vector<uint32_t> seg_skip;               // stuffed bytes + restart markers removed from every chunk of the scan
    int64_t mcus() const { return (int64_t)mcus_x * mcus_y; }
};

struct JpParser {
    const uint8_t* d; size_t n;
    std::string why;
    int fail(int code, const char* fmt, ...) {
        char buf[256];
        va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
        why = buf;
        return code;
    }
    int u16(size_t p) const { return (d[p] << 8) | d[p + 1]; }
};

// EXIF orientation the way cv::imdecode reads it (ExifReader) from the TIFF structure t [m bytes]: the byte order ("II" little endian,
// anything else big endian), the 0x2A mark, IFD0, the first entry with tag 0x0112 and the 16-bit value at +8 of the entry.  Entries
// are read until one would leave the structure.  The PNG decoder reads its eXIf chunk with it.
inline int jp_tiff_orientation(const uint8_t* t, size_t m) {
    const bool le = m > 1 && t[0] == 'I' && t[1] == 'I';
    auto get16 = [&](size_t o, int& v) { if (o + 1 >= m) return false; v = le ? t[o] | (t[o + 1] << 8) : (t[o] << 8) | t[o + 1]; return true; };
    int mark = 0;
    if (!get16(2, mark) || mark != 0x2A || 4 + 3 >= m) return 1;
    const uint32_t ifd = le ? (uint32_t)t[4] | (uint32_t)t[5] << 8 | (uint32_t)t[6] << 16 | (uint32_t)t[7] << 24
                            : (uint32_t)t[4] << 24 | (uint32_t)t[5] << 16 | (uint32_t)t[6] << 8 | (uint32_t)t[7];
    int cnt = 0;
    if (!get16(ifd, cnt)) return 1;
    size_t o = (size_t)ifd + 2;
    for (int e = 0; e < cnt; ++e, o += 12) {
        int tag = 0, v = 0;
        if (!get16(o, tag)) return 1;
        if (tag == 0x0112) return get16(o + 8, v) && v >= 1 && v <= 8 ? v : 1;
    }
    return 1;
}

// The same from a JPEG's first APP1 segment, whose 6 leading bytes are skipped without looking at them.
inline int jp_exif_orientation(const uint8_t* a, size_t len) {
    if (len <= 6) return 1;
    return jp_tiff_orientation(a + 6, len - 6);
}

// Parses the file and walks its scan.  chunk = the unstuffing chunk size (bytes) seg_skip is counted in.  Returns JP_* with the
// reason in `why`.
inline int jp_parse(const uint8_t* data, size_t size, size_t chunk, JpImage& im, std::string& why) {
    JpParser p{data, size, std::string()};
    auto done = [&](int rc) { why = p.why; return rc; };
    if (!data || size < 4 || data[0] != 0xFF || data[1] != 0xD8) return done(p.fail(JP_INVALID, "not a JPEG file (no SOI marker)"));
    int16_t qraw[4][64]; bool qdef[4] = {false, false, false, false};
    bool hdef[8] = {false, false, false, false, false, false, false, false};
    int cid[3] = {0, 0, 0}, qsel[3] = {0, 0, 0};
    bool have_sof = false, jfif = false, adobe = false, app1 = false;
    int adobe_transform = -1;
    size_t i = 2;
    for (;;) {
        if (i >= size || data[i] != 0xFF) return done(p.fail(JP_INVALID, "expected a marker at byte %zu", i));
        while (i < size && data[i] == 0xFF) ++i;                                   // fill bytes
        if (i >= size) return done(p.fail(JP_INVALID, "file ends inside a marker"));
        const int m = data[i++];
        if (m == 0xD9) return done(p.fail(JP_INVALID, "EOI before the scan"));
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;                       // TEM, stray RSTn: no length
        if (i + 2 > size) return done(p.fail(JP_INVALID, "file ends inside a marker segment"));
        const size_t L = (size_t)p.u16(i);
        if (L < 2 || i + L > size) return done(p.fail(JP_INVALID, "marker 0x%02X: segment length %zu past the end of the file", m, L));
        const uint8_t* s = data + i + 2; const size_t sl = L - 2;
        i += L;
        if (m == 0xC0 || m == 0xC1) {
            if (have_sof) return done(p.fail(JP_INVALID, "two SOF markers"));
            have_sof = true;
            if (sl < 6) return done(p.fail(JP_INVALID, "short SOF segment"));
            if (s[0] != 8) return done(p.fail(JP_UNSUPPORTED, "%d-bit samples (only 8-bit JPEG is supported)", s[0]));
            im.H = (s[1] << 8) | s[2]; im.W = (s[3] << 8) | s[4]; im.ncomp = s[5];
            if (im.ncomp != 1 && im.ncomp != 3) return done(p.fail(JP_UNSUPPORTED, "%d components (1 or 3 are supported)", im.ncomp));
            if (im.W == 0 || im.H == 0) return done(p.fail(im.H == 0 ? JP_UNSUPPORTED : JP_INVALID, "image size %dx%d", im.W, im.H));
            if (sl < 6 + 3 * (size_t)im.ncomp) return done(p.fail(JP_INVALID, "short SOF segment"));
            for (int c = 0; c < im.ncomp; ++c) {
                cid[c] = s[6 + 3 * c]; im.hs[c] = s[7 + 3 * c] >> 4; im.vs[c] = s[7 + 3 * c] & 15; qsel[c] = s[8 + 3 * c];
                if (im.hs[c] < 1 || im.hs[c] > 4 || im.vs[c] < 1 || im.vs[c] > 4 || qsel[c] > 3)
                    return done(p.fail(JP_INVALID, "bad sampling factors or table selector in SOF"));
            }
        } else if (m == 0xC2 || m == 0xC3 || (m >= 0xC5 && m <= 0xC7) || (m >= 0xC9 && m <= 0xCB) || (m >= 0xCD && m <= 0xCF) || m == 0xCC) {
            return done(p.fail(JP_UNSUPPORTED, "SOF/DAC marker 0x%02X: progressive, lossless, hierarchical and arithmetic-coded JPEG are not supported", m));
        } else if (m == 0xC4) {
            size_t o = 0;
            while (o < sl) {
                if (o + 17 > sl) return done(p.fail(JP_INVALID, "short DHT segment"));
                const int tc = s[o] >> 4, th = s[o] & 15;
                if (tc > 1 || th > 3) return done(p.fail(JP_INVALID, "bad DHT table class / id"));
                uint8_t bits[17]; bits[0] = 0;
                int cnt = 0;
                for (int l = 1; l <= 16; ++l) { bits[l] = s[o + l]; cnt += bits[l]; }
                if (cnt > 256 || o + 17 + cnt > sl) return done(p.fail(JP_INVALID, "bad DHT symbol count"));
                if (!jm_build_huff(bits, s + o + 17, cnt, tc == 0, im.tabs[tc * 4 + th])) return done(p.fail(JP_INVALID, "bad Huffman table"));
                hdef[tc * 4 + th] = true;
                o += 17 + cnt;
            }
        } else if (m == 0xDB) {
            size_t o = 0;
            while (o < sl) {
                const int pq = s[o] >> 4, tq = s[o] & 15;
                if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > sl) return done(p.fail(JP_INVALID, "bad DQT segment"));
                for (int k = 0; k < 64; ++k)
                    qraw[tq][jm_natural(k)] = (int16_t)(pq ? (s[o + 1 + 2 * k] << 8) | s[o + 2 + 2 * k] : s[o + 1 + k]);
                qdef[tq] = true;
                o += 1 + 64 * (pq + 1);
            }
        } else if (m == 0xDD) {
            if (sl < 2) return done(p.fail(JP_INVALID, "short DRI segment"));
            im.restart = (s[0] << 8) | s[1];
        } else if (m == 0xE0) {
            if (sl >= 14 && !memcmp(s, "JFIF", 5)) jfif = true;
        } else if (m == 0xE1) {
            if (!app1) { app1 = true; im.orient = jp_exif_orientation(s, sl); }
        } else if (m == 0xEE) {
            if (sl >= 12 && !memcmp(s, "Adobe", 5)) { adobe = true; adobe_transform = s[11]; }
        } else if (m == 0xDA) {
            if (!have_sof) return done(p.fail(JP_INVALID, "SOS before SOF"));
            if (sl < 1) return done(p.fail(JP_INVALID, "short SOS segment"));
            const int ns = s[0];
            if (ns != im.ncomp) return done(p.fail(JP_UNSUPPORTED, "a scan of %d of %d components (multi-scan files are not supported)", ns, im.ncomp));
            if (sl < 4 + 2 * (size_t)ns) return done(p.fail(JP_INVALID, "short SOS segment"));
            int dsel[3], asel[3];
            for (int c = 0; c < ns; ++c) {
                if (s[1 + 2 * c] != cid[c]) return done(p.fail(JP_UNSUPPORTED, "scan components out of frame order"));
                dsel[c] = s[2 + 2 * c] >> 4; asel[c] = s[2 + 2 * c] & 15;
                if (dsel[c] > 3 || asel[c] > 3 || !hdef[dsel[c]] || !hdef[4 + asel[c]]) return done(p.fail(JP_INVALID, "scan uses an undefined Huffman table"));
                if (!qdef[qsel[c]]) return done(p.fail(JP_INVALID, "component uses an undefined quantisation table"));
            }
            const uint8_t* t = s + 1 + 2 * ns;
            if (t[0] != 0 || t[1] != 63 || t[2] != 0) return done(p.fail(JP_INVALID, "sequential scan with Ss=%d Se=%d Ah/Al=0x%02X", t[0], t[1], t[2]));
            if (im.ncomp == 3) {
                if (!jfif && adobe && adobe_transform == 0) return done(p.fail(JP_UNSUPPORTED, "RGB JPEG (Adobe transform 0)"));
                if (!jfif && !adobe && cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B') return done(p.fail(JP_UNSUPPORTED, "RGB JPEG (component ids R, G, B)"));
                if (im.hs[1] != 1 || im.vs[1] != 1 || im.hs[2] != 1 || im.vs[2] != 1)
                    return done(p.fail(JP_UNSUPPORTED, "chroma sampling %dx%d / %dx%d", im.hs[1], im.vs[1], im.hs[2], im.vs[2]));
                const int f = im.hs[0] * 10 + im.vs[0];
                if (f != 11 && f != 21 && f != 22 && f != 12 && f != 41) return done(p.fail(JP_UNSUPPORTED, "luma sampling %dx%d", im.hs[0], im.vs[0]));
                im.hmax = im.hs[0]; im.vmax = im.vs[0];
            } else {
                im.hs[0] = im.vs[0] = 1;                   // a single-component scan is non-interleaved whatever the SOF says
                im.hmax = im.vmax = 1;
            }
            im.mcus_x = (im.W + 8 * im.hmax - 1) / (8 * im.hmax);
            im.mcus_y = (im.H + 8 * im.vmax - 1) / (8 * im.vmax);
            int b = 0;
            for (int c = 0; c < im.ncomp; ++c) {
                im.cw[c] = (int)(((int64_t)im.W * im.hs[c] + im.hmax - 1) / im.hmax);
                im.ch[c] = (int)(((int64_t)im.H * im.vs[c] + im.vmax - 1) / im.vmax);
                im.wb[c] = im.mcus_x * im.hs[c]; im.hb[c] = im.mcus_y * im.vs[c];
                for (int k = 0; k < 64; ++k) im.qt[c][k] = qraw[qsel[c]][k];
                for (int dy = 0; dy < im.vs[c]; ++dy)
                    for (int dx = 0; dx < im.hs[c]; ++dx, ++b) {
                        im.scan.blk_comp[b] = (uint8_t)c; im.scan.blk_dx[b] = (uint8_t)dx; im.scan.blk_dy[b] = (uint8_t)dy;
                        im.scan.dc_tab[b] = (int16_t)dsel[c]; im.scan.ac_tab[b] = (int16_t)(4 + asel[c]);
                    }
            }
            im.scan.bpm = b;
            const bool tr = im.orient >= 5;
            im.OW = tr ? im.H : im.W; im.OH = tr ? im.W : im.H;
            im.scan_off = i;
            break;
        }
        // every other marker segment (APPn, COM, DNL, ...) is skipped
    }
    // walk the entropy-coded data: stuffed zeros and restart markers are counted per chunk, the scan ends at the first other marker
    const size_t s0 = im.scan_off;
    const int64_t nseg = im.restart ? (im.mcus() + im.restart - 1) / im.restart : 1;
    im.seg_bytes.clear(); im.seg_skip.clear();
    size_t q = s0, seg0 = s0, seg_removed = 0;
    auto skip = [&](size_t pos) {
        const size_t c = (pos - s0) / chunk;
        if (im.seg_skip.size() <= c) im.seg_skip.resize(c + 1, 0);
        im.seg_skip[c]++;
    };
    for (;;) {
        const uint8_t* f = q < size ? (const uint8_t*)memchr(data + q, 0xFF, size - q) : nullptr;
        if (!f || (size_t)(f - data) + 1 >= size) return done(p.fail(JP_INVALID, "entropy-coded data runs to the end of the file (truncated)"));
        const size_t r = (size_t)(f - data);
        const int b = data[r + 1];
        if (b == 0) { skip(r + 1); ++seg_removed; q = r + 2; continue; }
        if (b >= 0xD0 && b <= 0xD7) {
            const int64_t k = (int64_t)im.seg_bytes.size();
            if (!im.restart || k + 1 >= nseg || b - 0xD0 != (int)(k & 7))
                return done(p.fail(JP_INVALID, "unexpected restart marker RST%d after segment %lld", b - 0xD0, (long long)k));
            im.seg_bytes.push_back((uint32_t)(r - seg0 - seg_removed));
            skip(r); skip(r + 1);
            seg0 = q = r + 2; seg_removed = 0;
            continue;
        }
        im.seg_bytes.push_back((uint32_t)(r - seg0 - seg_removed));
        im.scan_len = r - s0;
        break;
    }
    if ((int64_t)im.seg_bytes.size() != nseg)
        return done(p.fail(JP_INVALID, "%zu restart segments, %lld expected (missing restart markers)", im.seg_bytes.size(), (long long)nseg));
    im.seg_skip.resize((im.scan_len + chunk - 1) / chunk, 0);
    return done(JP_OK);
}
