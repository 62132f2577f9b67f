// tests/host_jpeg.cpp -- TEST HARNESS: runs the JPEG decoder's host parser (csrc/jpeg_parse.h) and its __host__ __device__ arithmetic
// (csrc/jpeg_math.cuh) on the CPU.  Two ways to get the coefficient blocks: the serial decoder (one MCU after the other), and the
// self-synchronising subsequence decode in the order csrc/jpeg.cu runs it (round 0 from guessed states, JD_ROUNDS parallel rounds
// -- here against a snapshot of the previous round --, the in-order sweep, the block prefix sum, the write pass).  Then the same DC
// prediction, IDCT, upsampling, colour conversion and orientation.  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/jpeg_parse.h"
#include <algorithm>
#include <vector>

namespace {

const int kRounds = 6;           // JD_ROUNDS: the parallel rounds jpeg.cu runs before its sweep

struct Seg { uint32_t b0, b1; int64_t first_mcu, n_mcu; };

struct WriteSink {
    int16_t* blocks; const JpImage* im; const Seg* sg; int64_t base; int64_t expected; bool* bad;
    // block ordinal `o` of the segment -> coefficient block
    int16_t* block(int64_t o) {
        const int bpm = im->scan.bpm;
        const int64_t m = sg->first_mcu + o / bpm; const int b = (int)(o % bpm);
        const int c = im->scan.blk_comp[b];
        const int64_t bx = (m % im->mcus_x) * im->hs[c] + im->scan.blk_dx[b], by = (m / im->mcus_x) * im->vs[c] + im->scan.blk_dy[b];
        int64_t off = 0;
        for (int cc = 0; cc < c; ++cc) off += (int64_t)im->wb[cc] * im->hb[cc];
        return blocks + 64 * (off + by * im->wb[c] + bx);
    }
    void coef(int ord, int k, int v) {
        const int64_t o = base + ord;
        if (o < 0) { *bad = true; return; }
        if (o < expected) block(o)[jm_natural(k)] = (int16_t)v;
    }
    void fail(int ord, int) { if (base + ord < expected) *bad = true; }
};

int64_t total_blocks(const JpImage& im) {
    int64_t t = 0;
    for (int c = 0; c < im.ncomp; ++c) t += (int64_t)im.wb[c] * im.hb[c];
    return t;
}

// unstuffed data (8 zero bytes of padding) and segment bit ranges, from the parser's walk
void unstuff(const uint8_t* d, const JpImage& im, std::vector<uint8_t>& u, std::vector<Seg>& segs) {
    u.clear();
    const uint8_t* s = d + im.scan_off;
    for (size_t i = 0; i < im.scan_len; ++i) {
        const uint8_t prev = i ? s[i - 1] : 0, b = s[i], next = i + 1 < im.scan_len ? s[i + 1] : 0;
        if (prev == 0xFF && (b == 0 || (b >= 0xD0 && b <= 0xD7))) continue;
        if (b == 0xFF && next >= 0xD0 && next <= 0xD7) continue;
        u.push_back(b);
    }
    u.resize(u.size() + 8, 0);
    segs.clear();
    uint32_t pos = 0;
    const int64_t R = im.restart ? im.restart : im.mcus();
    for (size_t k = 0; k < im.seg_bytes.size(); ++k) {
        Seg g; g.b0 = pos * 8; pos += im.seg_bytes[k]; g.b1 = pos * 8;
        g.first_mcu = (int64_t)k * R; g.n_mcu = std::min<int64_t>(R, im.mcus() - g.first_mcu);
        segs.push_back(g);
    }
}

bool decode_serial(const uint8_t* u, const JpImage& im, const std::vector<Seg>& segs, int16_t* coef, int64_t* stats) {
    bool bad = false;
    for (const Seg& sg : segs) {
        WriteSink sink{coef, &im, &sg, 0, sg.n_mcu * im.scan.bpm, &bad};
        uint32_t p = sg.b0;
        for (int64_t o = 0; o < sink.expected; ++o) {
            const int b = (int)(o % im.scan.bpm);
            int zz = 0;
            while (zz < 64) {
                const JmHuff& h = im.tabs[zz == 0 ? im.scan.dc_tab[b] : im.scan.ac_tab[b]];
                int k, v;
                if (!jm_step(u, p, sg.b1, h, zz, k, v)) return false;
                stats[0]++;
                if (k >= 0) sink.block(o)[jm_natural(k)] = (int16_t)v;
            }
        }
    }
    return !bad;
}

bool decode_subsequences(const uint8_t* u, const JpImage& im, const std::vector<Seg>& segs, uint32_t S, int16_t* coef, int64_t* stats) {
    bool bad = false;
    JmNoSink none;
    for (const Seg& sg : segs) {
        const uint32_t bits = sg.b1 - sg.b0;
        const int n = std::max<int>(1, (int)((bits + S - 1) / S));
        auto start = [&](int j) { return sg.b0 + (uint32_t)j * S; };
        auto stop = [&](int j) { return j + 1 == n ? sg.b1 : start(j + 1); };
        std::vector<uint64_t> ex(n);
        std::vector<int> computed(n, 0), changed(n, 0);
        int cw = 0;
        auto span = [&](int j, uint64_t entry, int* count) {
            return jm_span(u, jm_exit_pos(entry), jm_exit_state(entry), stop(j), sg.b1, im.scan, im.tabs, none, count);
        };
        for (int j = 0; j < n; ++j) ex[j] = span(j, jm_pack_exit(start(j), 0, 0), &cw);       // round 0
        stats[0] += cw; cw = 0;
        for (int r = 1; r <= kRounds; ++r) {
            const std::vector<uint64_t> prev = ex; const std::vector<int> prev_changed = changed;
            for (int j = 1; j < n; ++j) {
                if (prev_changed[j - 1] < computed[j]) continue;
                const uint64_t e = span(j, prev[j - 1], &cw);
                computed[j] = r;
                if (!jm_exit_same(e, ex[j])) changed[j] = r;
                ex[j] = e;
            }
            if (r <= 2) for (int j = 1; j < n; ++j) stats[2 + r] += changed[j] == r;
        }
        for (int j = 1; j < n; ++j) {                                                          // the sweep
            if (changed[j - 1] < computed[j]) continue;
            const uint64_t e = span(j, ex[j - 1], &cw);
            computed[j] = kRounds + 1;
            if (!jm_exit_same(e, ex[j])) changed[j] = kRounds + 1;
            ex[j] = e;
            stats[5]++;
        }
        stats[1] += cw; stats[2] += n;
        int64_t base = 0;
        const int64_t expected = sg.n_mcu * im.scan.bpm;
        for (int j = 0; j < n; ++j) {                                                          // the write pass
            WriteSink sink{coef, &im, &sg, base, expected, &bad};
            const uint64_t entry = j ? ex[j - 1] : jm_pack_exit(sg.b0, 0, 0);
            jm_span(u, jm_exit_pos(entry), jm_exit_state(entry), stop(j), sg.b1, im.scan, im.tabs, sink);
            base += jm_exit_nblk(ex[j]);
        }
        if (base < expected) bad = true;
    }
    return !bad;
}

void resolve_dc(const JpImage& im, const std::vector<Seg>& segs, int16_t* coef) {
    for (const Seg& sg : segs) {
        uint16_t run[3] = {0, 0, 0};
        WriteSink at{coef, &im, &sg, 0, 0, nullptr};
        for (int64_t o = 0; o < sg.n_mcu * im.scan.bpm; ++o) {
            int16_t* b = at.block(o);
            const int c = im.scan.blk_comp[o % im.scan.bpm];
            run[c] = (uint16_t)(run[c] + (uint16_t)b[0]);
            b[0] = (int16_t)run[c];
        }
    }
}

void reconstruct(const JpImage& im, const int16_t* coef, uint8_t* out) {
    std::vector<std::vector<uint8_t>> pl(im.ncomp);
    int64_t off = 0;
    for (int c = 0; c < im.ncomp; ++c) {
        const int stride = im.wb[c] * 8;
        pl[c].assign((size_t)stride * im.hb[c] * 8, 0);
        for (int by = 0; by < im.hb[c]; ++by)
            for (int bx = 0; bx < im.wb[c]; ++bx) {
                const int16_t* blk = coef + 64 * (off + (int64_t)by * im.wb[c] + bx);
                int ws[64];
                for (int col = 0; col < 8; ++col) jm_idct_col(blk, im.qt[c], col, ws);
                for (int r = 0; r < 8; ++r) jm_idct_row(ws, r, &pl[c][(size_t)(by * 8 + r) * stride + bx * 8]);
            }
        off += (int64_t)im.wb[c] * im.hb[c];
    }
    for (int oy = 0; oy < im.OH; ++oy)
        for (int ox = 0; ox < im.OW; ++ox) {
            int x, y;
            jm_orient_src(im.orient, im.W, im.H, ox, oy, x, y);
            uint8_t* o = out + ((size_t)oy * im.OW + ox) * 3;
            const int Y = pl[0][(size_t)y * im.wb[0] * 8 + x];
            if (im.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; continue; }
            int cc[2];
            for (int c = 1; c < 3; ++c)
                cc[c - 1] = jm_chroma(pl[c].data(), im.wb[c] * 8, im.cw[c], im.ch[c], im.hmax / im.hs[c], im.vmax / im.vs[c], x, y);
            jm_ycc_to_bgr(Y, cc[0], cc[1], o);
        }
}

}  // namespace

extern "C" {
// info[6] = W, H, output width, output height, components, coefficient blocks; returns the JP_* status
int hj_info(const uint8_t* d, size_t n, int64_t* info) {
    JpImage im; std::string why;
    const int rc = jp_parse(d, n, 4096, im, why);
    if (rc) return rc;
    info[0] = im.W; info[1] = im.H; info[2] = im.OW; info[3] = im.OH; info[4] = im.ncomp; info[5] = total_blocks(im);
    return 0;
}

// S == 0: serial decode; S > 0: subsequences of S bits.  out [OH*OW*3] and coef [blocks*64] (DC resolved) may be NULL.
// stats[6] = codewords of the first decode (serial: all; subsequences: round 0), codewords of the later rounds and the sweep,
// subsequences, subsequences whose exit changed in round 1 / in round 2, subsequences the sweep re-decoded.
int hj_decode(const uint8_t* d, size_t n, uint32_t S, uint8_t* out, int16_t* coef_out, int64_t* stats) {
    JpImage im; std::string why;
    const int rc = jp_parse(d, n, 4096, im, why);
    if (rc) return rc;
    std::vector<uint8_t> u; std::vector<Seg> segs;
    unstuff(d, im, u, segs);
    std::vector<int16_t> coef((size_t)total_blocks(im) * 64, 0);
    int64_t st[6] = {0, 0, 0, 0, 0, 0};
    const bool ok = S ? decode_subsequences(u.data(), im, segs, S, coef.data(), st) : decode_serial(u.data(), im, segs, coef.data(), st);
    if (stats) for (int i = 0; i < 6; ++i) stats[i] = st[i];
    if (!ok) return JP_INVALID;
    resolve_dc(im, segs, coef.data());
    if (coef_out) std::copy(coef.begin(), coef.end(), coef_out);
    if (out) reconstruct(im, coef.data(), out);
    return JP_OK;
}
}
