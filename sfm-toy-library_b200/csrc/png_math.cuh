// png_math.cuh -- arithmetic of the PNG decoder (csrc/png.cu) that the device and the host harness (tests/host_png.cpp) share:
// the deflate bit reader, canonical Huffman codes with zlib's acceptance rules, the block header and body decoders, the PNG filters
// and the sample unpacking of the colour stage.  __host__ __device__ when compiled by nvcc, plain inline C++ under g++.
#pragma once
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define PM_HD __host__ __device__ __forceinline__
#else
#define PM_HD inline
#endif

// Deflate bit reader, LSB first, fed 32 bits at a time from aligned words.  `d` must be 4-byte aligned and stay readable 16 bytes past
// `end_bit / 8` (the refill reads ahead); a position past `end_bit` is an overrun the caller checks with over().  After refill() at
// least 33 bits are buffered: a literal/length code with its extra bits, or a distance code with its extra bits.
struct PmBits {
    const uint8_t* d; uint64_t end_bit;
    uint64_t next;                // next byte to load into buf (a multiple of 4)
    uint64_t buf; int cnt;        // cnt valid bits in buf
    PM_HD uint32_t load32(uint64_t o) const {
#if defined(__CUDA_ARCH__)
        return __ldg((const unsigned int*)(d + o));
#else
        uint32_t v;
        memcpy(&v, d + o, 4);
        return v;                 // little-endian hosts
#endif
    }
    PM_HD void init(const uint8_t* data, uint64_t start_bit, uint64_t end) {
        d = data; end_bit = end; next = (start_bit >> 5) << 2; buf = 0; cnt = 0;
        refill(); refill();
        drop((int)(start_bit & 31));
    }
    PM_HD void refill() {
        if (cnt <= 32) { buf |= (uint64_t)load32(next) << cnt; next += 4; cnt += 32; }
    }
    PM_HD uint32_t peek(int n) const { return (uint32_t)(buf & ((1ull << n) - 1)); }
    PM_HD void drop(int n) { buf >>= n; cnt -= n; }
    PM_HD uint32_t get(int n) { const uint32_t v = peek(n); drop(n); return v; }   // n <= cnt
    PM_HD uint64_t pos() const { return next * 8 - (uint64_t)cnt; }
    PM_HD bool over() const { return pos() > end_bit; }
    PM_HD void align() { drop(cnt & 7); }
};

// Canonical Huffman code of deflate: a FAST-bit lookup table ((length << 9) | symbol, 0 = longer or unassigned code) and the
// count / sorted-symbol arrays of the canonical decode for the rest.
template <int FAST, int NSYM>
struct PmHuff {
    uint16_t fast[1 << FAST];
    uint16_t count[16];
    uint16_t sym[NSYM];
    // zlib's inflate_table: an over-subscribed code fails; an incomplete one fails unless `allow_single` (literal/length and distance
    // codes) and its longest length is 1.  An empty code is accepted here; decoding from it fails.
    PM_HD bool build(const uint8_t* len, int n, bool allow_single) {
        for (int l = 0; l < 16; ++l) count[l] = 0;
        for (int s = 0; s < n; ++s) count[len[s]]++;
        int max = 15;
        while (max > 0 && count[max] == 0) --max;
        int left = 1;
        for (int l = 1; l <= 15; ++l) { left <<= 1; left -= count[l]; if (left < 0) return false; }
        if (max > 0 && left > 0 && (!allow_single || max != 1)) return false;
        uint16_t offs[16];
        offs[1] = 0;
        for (int l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + count[l]);
        for (int s = 0; s < n; ++s) if (len[s]) sym[offs[len[s]]++] = (uint16_t)s;
        for (int i = 0; i < (1 << FAST); ++i) fast[i] = 0;
        uint32_t code = 0;
        int k = 0;
        for (int l = 1; l <= 15; ++l) {
            for (int c = 0; c < count[l]; ++c, ++k, ++code) {
                if (l > FAST) continue;
                uint32_t rev = 0;
                for (int b = 0; b < l; ++b) rev |= ((code >> b) & 1u) << (l - 1 - b);
                for (uint32_t r = rev; r < (1u << FAST); r += 1u << l) fast[r] = (uint16_t)((l << 9) | sym[k]);
            }
            code <<= 1;
        }
        return true;
    }
    // the next symbol, or -1 for an unassigned code; needs 15 valid bits in b
    PM_HD int decode(PmBits& b) const {
        const uint32_t e = fast[b.peek(FAST)];
        if (e) { b.drop((int)(e >> 9)); return (int)(e & 511); }
        const uint32_t bits = b.peek(15);
        int code = 0, first = 0, index = 0;
        for (int l = 1; l <= 15; ++l) {
            code |= (int)((bits >> (l - 1)) & 1u);
            const int c = count[l];
            if (code - c < first) { b.drop(l); return sym[index + (code - first)]; }
            index += c; first += c; first <<= 1; code <<= 1;
        }
        return -1;
    }
};
typedef PmHuff<9, 288> PmLit;
typedef PmHuff<8, 32> PmDist;
typedef PmHuff<7, 19> PmCl;

// Block types and decode results
enum { PM_STORED = 0, PM_FIXED = 1, PM_DYNAMIC = 2 };
enum { PM_OK = 0, PM_BAD = 1, PM_OVERRUN = 2, PM_FAR = 3, PM_STOP = 4 };   // FAR: a distance before the start; STOP: the sink quit

// deflate's length and distance bases as formulas (a table would be rebuilt in local memory on every call on the device)
PM_HD int pm_len_base(int s) { return s < 8 ? 3 + s : s == 28 ? 258 : ((4 + (s & 3)) << ((s - 4) >> 2)) + 3; }
PM_HD int pm_len_extra(int s) { return s < 8 || s == 28 ? 0 : (s - 4) >> 2; }
PM_HD int pm_dist_base(int s) { return s < 4 ? 1 + s : ((2 + (s & 1)) << ((s - 2) >> 1)) + 1; }
PM_HD int pm_dist_extra(int s) { return s < 4 ? 0 : (s - 2) >> 1; }

PM_HD void pm_fixed_tables(PmLit& lit, PmDist& dist) {
    uint8_t l[288];
    for (int s = 0; s < 288; ++s) l[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
    lit.build(l, 288, true);
    for (int s = 0; s < 30; ++s) l[s] = 5;
    l[30] = l[31] = 5;
    dist.build(l, 32, true);
}

// The dynamic-Huffman header after BFINAL and BTYPE, with zlib's checks: HLIT <= 286, HDIST <= 30, a complete code-length code,
// lengths that fill exactly HLIT + HDIST entries (a repeat with nothing before it or past the end fails), a non-zero end-of-block
// length, and literal/length and distance codes inflate_table accepts.
PM_HD bool pm_dynamic_header(PmBits& b, PmLit& lit, PmDist& dist) {
    b.refill();
    const int nlen = (int)b.get(5) + 257, ndist = (int)b.get(5) + 1, ncode = (int)b.get(4) + 4;
    if (nlen > 286 || ndist > 30) return false;
    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint8_t cl[19];
    for (int i = 0; i < 19; ++i) cl[i] = 0;
    for (int i = 0; i < ncode; ++i) { if (b.cnt < 3) b.refill(); cl[order[i]] = (uint8_t)b.get(3); }
    PmCl clc;
    if (!clc.build(cl, 19, false)) return false;
    if (clc.count[0] == 19) return false;                 // an empty code-length code decodes nothing but zeros: no end-of-block
    uint8_t lens[316];
    int have = 0;
    while (have < nlen + ndist) {
        b.refill();
        if (b.over()) return false;
        const int s = clc.decode(b);
        if (s < 0) return false;
        if (s < 16) { lens[have++] = (uint8_t)s; continue; }
        int rep, val = 0;
        if (s == 16) { if (have == 0) return false; val = lens[have - 1]; rep = 3 + (int)b.get(2); }
        else if (s == 17) rep = 3 + (int)b.get(3);
        else rep = 11 + (int)b.get(7);
        if (have + rep > nlen + ndist) return false;
        while (rep--) lens[have++] = (uint8_t)val;
    }
    if (lens[256] == 0) return false;
    if (!lit.build(lens, nlen, true)) return false;
    if (!dist.build(lens + nlen, ndist, true)) return false;
    return !b.over();
}

// Decodes one block body up to and including its end-of-block code.  The sink sees lit(byte) and copy(distance, length); its
// copy may refuse a distance (returns false: PM_FAR) and its lit may stop the decode (returns false: PM_STOP).  Returns PM_OK, PM_BAD
// (an unassigned or invalid code), PM_OVERRUN, PM_FAR or PM_STOP.
template <class Sink>
PM_HD int pm_huff_body(PmBits& b, const PmLit& lit, const PmDist& dist, Sink& s) {
    for (;;) {
        b.refill();
        if (b.over()) return PM_OVERRUN;
        const int sym = lit.decode(b);
        if (sym < 0) return PM_BAD;
        if (sym < 256) { if (!s.lit((uint32_t)sym)) return PM_STOP; continue; }
        if (sym == 256) return b.over() ? PM_OVERRUN : PM_OK;
        const int ls = sym - 257;
        if (ls >= 29) return PM_BAD;
        const int len = pm_len_base(ls) + (int)b.get(pm_len_extra(ls));
        b.refill();
        const int ds = dist.decode(b);
        if (ds < 0 || ds >= 30) return PM_BAD;
        const uint32_t d = (uint32_t)pm_dist_base(ds) + b.get(pm_dist_extra(ds));
        if (!s.copy(d, (uint32_t)len)) return PM_FAR;
    }
}

// A stored block after its 3 header bits: aligns, checks LEN / NLEN and hands the bytes to the sink.  The reader is left after them.
template <class Sink>
PM_HD int pm_stored_body(PmBits& b, Sink& s) {
    b.align();
    b.refill();
    const uint32_t len = b.get(16), nlen = b.get(16);   // 32 bits: cnt >= 33 after the refill
    if ((len ^ 0xffffu) != nlen) return PM_BAD;
    const uint64_t p = b.pos();
    if (p + 8ull * len > b.end_bit) return PM_OVERRUN;
    s.stored(b.d + (p >> 3), len);
    b.init(b.d, p + 8ull * len, b.end_bit);
    return PM_OK;
}

// ---------------------------------------------------------------------------------------------------------------- speculation
// A dynamic-Huffman block may start at bit p of d (zbits bits): BTYPE 2 and a header zlib accepts.  BFINAL may be either.
PM_HD bool pm_candidate(const uint8_t* d, uint64_t p, uint64_t zbits, PmLit& lit, PmDist& dist) {
    if (p + 17 > zbits) return false;
    PmBits b;
    b.init(d, p, zbits);
    if (((b.buf >> 1) & 3) != 2) return false;
    const uint32_t hlit = (uint32_t)(b.buf >> 3) & 31, hdist = (uint32_t)(b.buf >> 8) & 31;
    if (hlit > 29 || hdist > 29) return false;
    b.drop(3);
    return pm_dynamic_header(b, lit, dist);
}

struct PmProbeSink {          // counts output bytes and symbols; gives up past `cap` symbols
    uint64_t n = 0; uint32_t syms = 0, cap = 0;
    PM_HD bool lit(uint32_t) { ++n; return ++syms <= cap; }
    PM_HD bool copy(uint32_t, uint32_t len) { n += len; return ++syms <= cap; }
    PM_HD void stored(const uint8_t*, uint32_t len) { n += len; }
};

// Decodes the candidate block at p to its end-of-block: true with its end bit and output byte count, false if it is not a block
// (an invalid code, an overrun, or more than `cap` symbols).  Distances are not checked: the block's output position is not known yet.
PM_HD bool pm_probe(const uint8_t* d, uint64_t p, uint64_t zbits, uint32_t cap, PmLit& lit, PmDist& dist, uint64_t* end, uint64_t* n) {
    PmBits b;
    b.init(d, p, zbits);
    b.drop(3);
    if (!pm_dynamic_header(b, lit, dist)) return false;
    PmProbeSink s;
    s.cap = cap;
    if (pm_huff_body(b, lit, dist, s) != PM_OK) return false;
    *end = b.pos(); *n = s.n;
    return true;
}

// Sink that only counts output bytes (the chain's own decode and the probe)
struct PmCount {
    uint64_t n = 0;
    PM_HD bool lit(uint32_t) { ++n; return true; }
    PM_HD bool copy(uint32_t, uint32_t len) { n += len; return true; }
    PM_HD void stored(const uint8_t*, uint32_t len) { n += len; }
};

// ---------------------------------------------------------------------------------------------------------------- filters, colour
PM_HD int pm_paeth(int a, int b, int c) {
    const int p = a + b - c;
    int pa = p - a, pb = p - b, pc = p - c;
    pa = pa < 0 ? -pa : pa; pb = pb < 0 ? -pb : pb; pc = pc < 0 ? -pc : pc;
    return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}
// reconstructed byte of filter type f from the filtered byte x, left a, up b, upper-left c
PM_HD uint8_t pm_unfilter(int f, int x, int a, int b, int c) {
    switch (f) {
    case 1: return (uint8_t)(x + a);
    case 2: return (uint8_t)(x + b);
    case 3: return (uint8_t)(x + ((a + b) >> 1));
    case 4: return (uint8_t)(x + pm_paeth(a, b, c));
    default: return (uint8_t)x;
    }
}

// Adam7: pass p's first column / row and steps
PM_HD int pm_a7_x0(int p) { return p == 1 ? 4 : p == 3 ? 2 : p == 5 ? 1 : 0; }
PM_HD int pm_a7_y0(int p) { return p == 2 ? 4 : p == 4 ? 2 : p == 6 ? 1 : 0; }
PM_HD int pm_a7_dx(int p) { return p <= 1 ? 8 : p <= 3 ? 4 : p <= 5 ? 2 : 1; }
PM_HD int pm_a7_dy(int p) { return p <= 2 ? 8 : p <= 4 ? 4 : 2; }
// the pass pixel (x, y) belongs to
PM_HD int pm_a7_pass(int x, int y) {
    if (y & 1) return 6;
    if (x & 1) return 5;
    if (y & 2) return 4;
    if (x & 2) return 3;
    if (y & 4) return 2;
    if (x & 4) return 1;
    return 0;
}

// Sample k (0-based, in row order) of a reconstructed row at bit depth bd, as libpng leaves it for cv::imread: 16-bit samples keep their
// high byte; sub-byte grey is scaled to 8 bits (v * 255 / (2^bd - 1)) unless it is a palette index (`index`).
PM_HD int pm_sample(const uint8_t* row, int64_t k, int bd, bool index) {
    if (bd == 8) return row[k];
    if (bd == 16) return row[2 * k];
    const int64_t bit = k * bd;
    const int v = (row[bit >> 3] >> (8 - bd - (int)(bit & 7))) & ((1 << bd) - 1);
    if (index) return v;
    return bd == 1 ? v * 255 : bd == 2 ? v * 85 : v * 17;
}
