// tests/host_png.cpp -- TEST HARNESS: runs the PNG decoder's host parser (csrc/png_parse.h) and its __host__ __device__ arithmetic
// (csrc/png_math.cuh) on the CPU, in the order csrc/png.cu runs it: the scan for dynamic block headers and the probe of every
// candidate, the in-order block chain that takes a probed block wherever one starts at its position, every block decoded again into one word
// per output byte (here in reverse block order, to show that blocks do not depend on each other's words), the pointer-jumping rounds
// (here against a snapshot of the previous round), the Adler-32 check, the unfilter and the colour stage.  Also a plain serial
// inflate and the dynamic-header test alone.  Not part of the product library.
#include "../sfm-toy-library_b200/csrc/png_parse.h"
#include <vector>

namespace {

const uint32_t kLit = 0x80000000u;

struct Count {
    uint64_t n = 0;
    bool lit(uint32_t) { ++n; return true; }
    bool copy(uint32_t d, uint32_t len) { if (d > n) return false; n += len; return true; }
    void stored(const uint8_t*, uint32_t len) { n += len; }
};
struct Words {
    uint32_t* w; uint64_t pos, blk, raw;
    void put(uint32_t v) { if (pos < raw) w[pos] = v; ++pos; }
    bool lit(uint32_t v) { put(kLit | v); return true; }
    bool copy(uint32_t d, uint32_t len) {
        if (d > pos) return false;
        for (uint32_t k = 0; k < len; ++k) { const uint64_t s = pos - d; put(pos >= raw ? 0 : s >= blk ? w[s] : (uint32_t)s); }
        return true;
    }
    void stored(const uint8_t* p, uint32_t len) { for (uint32_t k = 0; k < len; ++k) put(kLit | p[k]); }
};
struct Bytes {
    std::vector<uint8_t>* o;
    bool lit(uint32_t v) { o->push_back((uint8_t)v); return true; }
    bool copy(uint32_t d, uint32_t len) {
        if (d > o->size()) return false;
        for (uint32_t k = 0; k < len; ++k) o->push_back((*o)[o->size() - d]);
        return true;
    }
    void stored(const uint8_t* p, uint32_t len) { o->insert(o->end(), p, p + len); }
};

template <class Sink>
int block(PmBits& b, PmLit& lit, PmDist& dist, Sink& s, int* final, int* type) {
    b.refill();
    *final = (int)b.get(1); *type = (int)b.get(2);
    if (*type == PM_STORED) return pm_stored_body(b, s);
    if (*type == PM_FIXED) { pm_fixed_tables(lit, dist); return pm_huff_body(b, lit, dist, s); }
    if (*type == PM_DYNAMIC) return pm_dynamic_header(b, lit, dist) ? pm_huff_body(b, lit, dist, s) : PM_BAD;
    return PM_BAD;
}

}  // namespace

extern "C" {

// serial inflate of a zlib stream (header skipped, no Adler check): 0 and the bytes, or the PM_* failure
int hp_inflate(const uint8_t* z, size_t zlen, uint8_t* out, size_t cap, size_t* outlen, int64_t* nblocks) {
    std::vector<uint8_t> pad(z, z + zlen); pad.resize(zlen + 32, 0);
    std::vector<uint8_t> o;
    PmLit lit; PmDist dist;
    PmBits b; b.init(pad.data(), 16, (uint64_t)zlen * 8);
    Bytes s{&o};
    int final = 0, type = 0;
    *nblocks = 0;
    do {
        const int rc = block(b, lit, dist, s, &final, &type);
        ++*nblocks;
        if (rc) return rc;
    } while (!final);
    *outlen = o.size();
    if (o.size() > cap) return 9;
    memcpy(out, o.data(), o.size());
    return 0;
}

// 1 when a dynamic-Huffman header (after BFINAL / BTYPE) at bit `bit` of d passes zlib's checks
int hp_dynamic_header(const uint8_t* d, size_t len, uint64_t bit) {
    std::vector<uint8_t> pad(d, d + len); pad.resize(len + 32, 0);
    PmLit lit; PmDist dist;
    PmBits b; b.init(pad.data(), bit, (uint64_t)len * 8);
    return pm_dynamic_header(b, lit, dist) ? 1 : 0;
}

// info: format, OW, OH, W, H, orient, raw bytes, IDAT bytes
int hp_info(const uint8_t* data, size_t size, int64_t* info) {
    PgImage im; std::string why;
    const int rc = pg_parse(data, size, im, why);
    if (rc) return rc;
    info[0] = 2; info[1] = im.OW; info[2] = im.OH; info[3] = im.W; info[4] = im.H; info[5] = im.orient; info[6] = im.raw; info[7] = (int64_t)im.zlen;
    return 0;
}

// The decode in png.cu's order.  out: OW x OH x 3.  stats: blocks, stored, fixed, rounds.  Returns the SFMB200 status.
int hp_decode(const uint8_t* data, size_t size, uint8_t* out, int64_t* stats) {
    PgImage im; std::string why;
    if (int rc = pg_parse(data, size, im, why)) return rc;
    std::vector<uint8_t> z;
    for (auto& c : im.idat) z.insert(z.end(), data + c.first, data + c.first + c.second);
    const uint64_t zbits = (uint64_t)z.size() * 8;
    z.resize(z.size() + 32, 0);
    PmLit lit; PmDist dist;
    // scan (the first kCap candidates of every window of kWin bit offsets) and probe
    const int kWin = 512, kCap = 4;
    struct Cand { uint64_t bit, end, n; bool ok; };
    const uint64_t nwin = (zbits - 16) / kWin + 1;
    std::vector<std::vector<Cand>> win(nwin);
    for (uint64_t p = 16; p < zbits; ++p) {
        auto& v = win[(p - 16) / kWin];
        if (v.size() < (size_t)kCap && pm_candidate(z.data(), p, zbits, lit, dist)) v.push_back({p, 0, 0, false});
    }
    for (auto& v : win)
        for (auto& c : v) c.ok = pm_probe(z.data(), c.bit, zbits, 1u << 17, lit, dist, &c.end, &c.n);
    // chain
    struct Blk { uint64_t bit0, out0; };
    std::vector<Blk> blks;
    uint64_t pos = 16, outn = 0;
    int64_t stored = 0, fixed = 0, spec = 0;
    for (;;) {
        blks.push_back({pos, outn});
        PmBits b; b.init(z.data(), pos, zbits);
        const int bfinal = (int)(b.buf & 1);
        bool hit = false;
        if (((b.buf >> 1) & 3) == 2)
            for (auto& c : win[(pos - 16) / kWin])
                if (c.bit == pos && c.ok) { hit = true; pos = c.end; outn += c.n; break; }
        if (hit) { ++spec; if (bfinal) break; continue; }
        Count c; c.n = outn;
        int final = 0, type = 0;
        if (block(b, lit, dist, c, &final, &type)) return 1;
        stored += type == PM_STORED; fixed += type == PM_FIXED;
        pos = b.pos(); outn = c.n;
        if (final) break;
    }
    const uint64_t a = (pos + 7) >> 3;
    if (a + 4 > zbits / 8 || outn < (uint64_t)im.raw) return 1;
    const uint32_t adler = (uint32_t)z[a] << 24 | (uint32_t)z[a + 1] << 16 | (uint32_t)z[a + 2] << 8 | z[a + 3];
    // write, last block first
    std::vector<uint32_t> w((size_t)im.raw);
    for (size_t k = blks.size(); k-- > 0;) {
        if (blks[k].out0 >= (uint64_t)im.raw) continue;
        PmBits b; b.init(z.data(), blks[k].bit0, zbits);
        Words s{w.data(), blks[k].out0, blks[k].out0, (uint64_t)im.raw};
        int final = 0, type = 0;
        if (block(b, lit, dist, s, &final, &type)) return 1;         // a probed block's distances are checked here
    }
    // rounds against a snapshot
    int rounds = 0;
    for (;;) {
        ++rounds;
        const std::vector<uint32_t> prev = w;
        bool changed = false;
        for (size_t k = 0; k < w.size(); ++k)
            if (!(prev[k] & kLit)) { w[k] = prev[prev[k]]; changed = true; }
        if (!changed || rounds > 64) break;
    }
    std::vector<uint8_t> raw(w.size());
    uint64_t s1 = 0, s2 = 0;
    for (size_t k = 0; k < w.size(); ++k) {
        if (!(w[k] & kLit)) return 1;
        raw[k] = (uint8_t)w[k];
        s1 = (s1 + raw[k]) % 65521; s2 = (s2 + (uint64_t)((im.raw - (int64_t)k) % 65521) * raw[k]) % 65521;
    }
    if (outn == (uint64_t)im.raw) {
        const uint32_t A = (uint32_t)((1 + s1) % 65521), B = (uint32_t)(((uint64_t)im.raw % 65521 + s2) % 65521);
        if ((B << 16 | A) != adler) return 1;
    }
    // unfilter (row by row: the wavefront of png.cu computes the same recurrence)
    for (int p = 0; p < im.npass; ++p) {
        const int64_t rb = im.prow[p];
        for (int64_t r = 0; r < im.ph[p]; ++r) {
            uint8_t* row = raw.data() + im.poff[p] + r * (rb + 1);
            const int f = row[0];
            if (f > 4) return 1;
            for (int64_t x = 0; x < rb; ++x) {
                const int left = x >= im.bpp ? row[1 + x - im.bpp] : 0;
                const int up = r > 0 ? row[1 + x - (rb + 1)] : 0;
                const int ul = r > 0 && x >= im.bpp ? row[1 + x - im.bpp - (rb + 1)] : 0;
                row[1 + x] = pm_unfilter(f, row[1 + x], left, up, ul);
            }
        }
    }
    // colour
    for (int oy = 0; oy < im.OH; ++oy)
        for (int ox = 0; ox < im.OW; ++ox) {
            int x, y;
            jm_orient_src(im.orient, im.W, im.H, ox, oy, x, y);
            int p = 0, px = x, py = y;
            if (im.interlace) { p = pm_a7_pass(x, y); px = (x - pm_a7_x0(p)) / pm_a7_dx(p); py = (y - pm_a7_y0(p)) / pm_a7_dy(p); }
            const uint8_t* row = raw.data() + im.poff[p] + (int64_t)py * (im.prow[p] + 1) + 1;
            const int c = im.channels;
            int R, G, B;
            if (im.ct == 3) { const uint8_t* e = im.pal + 3 * pm_sample(row, px, im.bd, true); R = e[0]; G = e[1]; B = e[2]; }
            else if (c <= 2) R = G = B = pm_sample(row, (int64_t)px * c, im.bd, false);
            else { R = pm_sample(row, (int64_t)px * c, im.bd, false); G = pm_sample(row, (int64_t)px * c + 1, im.bd, false); B = pm_sample(row, (int64_t)px * c + 2, im.bd, false); }
            uint8_t* o = out + ((int64_t)oy * im.OW + ox) * 3;
            o[0] = (uint8_t)B; o[1] = (uint8_t)G; o[2] = (uint8_t)R;
        }
    if (stats) { stats[0] = (int64_t)blks.size(); stats[1] = stored; stats[2] = fixed; stats[3] = rounds; stats[4] = spec; }
    return 0;
}

}  // extern "C"
