// png.cu -- the PNG backend of the decode entry points (decode.cu checks a call and parses its files with png_parse.h): PNG files
// decoded on the device, byte-identical to cv::imread(IMREAD_COLOR) (include/sfmb200.h).
//
// The host packs the IDAT payloads of a group of images into one pinned buffer: one upload.  On the device, per group:
//   pg_scan       one thread per window of 512 bit offsets keeps the first 4 offsets where a dynamic-Huffman block header zlib accepts
//                 could start (HLIT, HDIST, a complete code-length code, the lengths, the literal/length and distance codes)
//   pg_probe      one thread per candidate decodes it to its end-of-block: end bit and output bytes, or not a block
//   pg_chain      one thread per image walks the true block sequence from the first block: where a probed candidate starts at its
//                 position it takes the candidate's end, otherwise (stored, fixed-Huffman, unprobed blocks) it decodes the block itself;
//                 it records every block's start bit and output offset, and the Adler-32 trailer
//   pg_write      one thread per block decodes it again from its recorded start into one 32-bit word per output byte: the byte itself,
//                 or, for a copy reaching before the block, the index of the byte it copies (copies inside the block resolve in place)
//   pg_round      pointer jumping: a word that points at a resolved word takes its byte, any other takes its source's source; a round
//                 returns at once when the round before changed nothing
//   pg_pack       the bytes out of the words, and the Adler-32 partial sums
//   pg_unfilter   one CTA per (image, Adam7 pass): a wavefront in which the thread of row r reconstructs pixel s - r at step s
//   pg_color      Adam7 scatter, sub-byte unpacking, palette, grey / alpha / 16-bit to B,G,R, and the EXIF orientation
//   rz_*          (scale != 1) the downscale of resize.cu
// then one download (per-image results and the images) and one host synchronisation.
#include "common.cuh"
#include "png_parse.h"
#include "resize_math.cuh"

#include <algorithm>

namespace {

constexpr int PG_THREADS = 16;           // decode threads per CTA: each keeps its Huffman tables in shared memory
constexpr int PG_ROUNDS = 32;            // resolution rounds launched (each hop crosses at least one block boundary)
constexpr uint32_t PG_LIT = 0x80000000u; // a word holding a resolved byte
constexpr int PG_WIN = 512;              // bits of the stream one scan thread tests
constexpr int PG_CAP = 4;                // candidates kept per window (the first ones)
constexpr uint32_t PG_PROBE_SYMS = 1u << 17;   // a probe gives up past this many symbols (zlib writes at most 2^15 - 1 per block)
constexpr uint32_t PG_NONE = 0xFFFFFFFFu;      // an empty candidate slot
enum { PG_E_DEFLATE = 1, PG_E_FAR = 2, PG_E_SHORT = 4, PG_E_TRUNC = 8, PG_E_ADLER = 16, PG_E_FILTER = 32, PG_E_BLOCKS = 64, PG_E_UNRESOLVED = 128 };

struct PgImg {
    long long z0, zbits;                 // the image's IDAT data in the upload (byte offset, length in bits)
    long long w0, raw;                   // its first word / raw byte in the group's arrays, and the raw size
    long long blk0, blkcap;              // its block records
    long long out0;                      // its decoded image (device memory of the group's images)
    long long pal0;                      // its palette in the upload
    long long win0, nwin;                // its scan windows (candidate slots win0 * PG_CAP ...)
    int W, H, OW, OH, orient, bd, ct, channels, bpp, npass, interlace, pad;
    long long pw[7], ph[7], prow[7], poff[7];
};
struct PgRes {                           // downloaded per image
    int err, nblocks, chain, stored, fixed, check_adler, spec, probed;
    unsigned adler, pad;
    unsigned long long out, s1, s2;
};
struct PgBlk { uint32_t bit0, out0; };
struct PgCand { uint32_t bit, end, n, ok; };     // a possible dynamic block start and, once probed, its end bit and output bytes

// the image whose [first, next first) range of some per-image index holds k (the last i with first(i) <= k)
template <class F>
__device__ __forceinline__ int pg_image_of(long long k, int n, F first) {
    int lo = 0, hi = n - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (first(mid) <= k) lo = mid; else hi = mid - 1; }
    return lo;
}

// ---------------------------------------------------------------------------------------------------------------- inflate
struct ChainSink {                       // counts output bytes and refuses a distance before the start of the stream
    unsigned long long n;
    __device__ bool lit(uint32_t) { ++n; return true; }
    __device__ bool copy(uint32_t d, uint32_t len) { if (d > n) return false; n += len; return true; }
    __device__ void stored(const uint8_t*, uint32_t len) { n += len; }
};

// One thread per window of PG_WIN bit offsets: the first PG_CAP offsets where a dynamic block header zlib accepts could start.
__global__ void __launch_bounds__(PG_THREADS) pg_scan(const uint8_t* __restrict__ z, const PgImg* __restrict__ imgs, int n, long long nwin,
                                                      PgCand* cands) {
    __shared__ PmLit s_lit[PG_THREADS];
    __shared__ PmDist s_dist[PG_THREADS];
    for (long long w = (long long)blockIdx.x * PG_THREADS + threadIdx.x; w < nwin; w += (long long)gridDim.x * PG_THREADS) {
        const PgImg& im = imgs[pg_image_of(w, n, [&](int i) { return imgs[i].win0; })];
        const uint8_t* d = z + im.z0;
        const uint64_t p0 = 16 + (uint64_t)(w - im.win0) * PG_WIN, p1 = min(p0 + PG_WIN, (uint64_t)im.zbits);
        int k = 0;
        for (uint64_t p = p0; p < p1 && k < PG_CAP; ++p)
            if (pm_candidate(d, p, (uint64_t)im.zbits, s_lit[threadIdx.x], s_dist[threadIdx.x])) cands[w * PG_CAP + k++] = PgCand{(uint32_t)p, 0, 0, 0};
    }
}

// One thread per candidate: decodes it to its end-of-block.
__global__ void __launch_bounds__(PG_THREADS) pg_probe(const uint8_t* __restrict__ z, const PgImg* __restrict__ imgs, int n, long long nslot,
                                                       PgCand* cands, PgRes* res) {
    __shared__ PmLit s_lit[PG_THREADS];
    __shared__ PmDist s_dist[PG_THREADS];
    for (long long q = (long long)blockIdx.x * PG_THREADS + threadIdx.x; q < nslot; q += (long long)gridDim.x * PG_THREADS) {
        PgCand c = cands[q];
        if (c.bit == PG_NONE) continue;
        const int i = pg_image_of(q / PG_CAP, n, [&](int j) { return imgs[j].win0; });
        const PgImg& im = imgs[i];
        uint64_t end = 0, cnt = 0;
        c.ok = pm_probe(z + im.z0, c.bit, (uint64_t)im.zbits, PG_PROBE_SYMS, s_lit[threadIdx.x], s_dist[threadIdx.x], &end, &cnt)
               && cnt < 0xFFFFFFFFull;
        c.end = (uint32_t)end; c.n = (uint32_t)cnt;
        cands[q] = c;
        atomicAdd(&res[i].probed, 1);
    }
}

__global__ void __launch_bounds__(PG_THREADS) pg_chain(const uint8_t* __restrict__ z, const PgImg* __restrict__ imgs, int n,
                                                       const PgCand* __restrict__ cands, PgBlk* blks, PgRes* res) {
    __shared__ PmLit s_lit[PG_THREADS];
    __shared__ PmDist s_dist[PG_THREADS];
    const int i = blockIdx.x * PG_THREADS + threadIdx.x;
    if (i >= n) return;
    const PgImg& im = imgs[i];
    PmLit& lit = s_lit[threadIdx.x];
    PmDist& dist = s_dist[threadIdx.x];
    const uint8_t* d = z + im.z0;
    unsigned long long pos = 16, out = 0;
    int nb = 0, err = 0, chain = 0, stored = 0, fixed = 0, spec = 0;
    for (;;) {
        if (nb >= im.blkcap) { err = PG_E_BLOCKS; break; }
        blks[im.blk0 + nb] = PgBlk{(uint32_t)pos, (uint32_t)min(out, 0xFFFFFFFFull)};
        ++nb;
        PmBits b;
        b.init(d, pos, (uint64_t)im.zbits);
        const int final = (int)b.get(1), type = (int)b.get(2);
        if (type == PM_DYNAMIC) {                                // a probed candidate starting here: take its end
            const long long w = (long long)(pos - 16) / PG_WIN;
            bool hit = false;
            for (int k = 0; k < PG_CAP && w < im.nwin && !hit; ++k) {
                const PgCand c = cands[(im.win0 + w) * PG_CAP + k];
                if (c.bit == pos && c.ok) { hit = true; pos = c.end; out += c.n; }
            }
            if (hit) { ++spec; if (final) break; continue; }
        }
        ChainSink s{out};
        int rc = PM_OK;
        if (type == PM_STORED) { rc = pm_stored_body(b, s); ++stored; }
        else if (type == PM_FIXED) { pm_fixed_tables(lit, dist); rc = pm_huff_body(b, lit, dist, s); ++fixed; }
        else if (type == PM_DYNAMIC) { rc = pm_dynamic_header(b, lit, dist) ? pm_huff_body(b, lit, dist, s) : PM_BAD; }
        else rc = PM_BAD;
        ++chain;
        if (rc != PM_OK) { err = rc == PM_FAR ? PG_E_FAR : rc == PM_OVERRUN ? PG_E_TRUNC : PG_E_DEFLATE; break; }
        pos = b.pos(); out = s.n;
        if (final) break;
    }
    PgRes& r = res[i];
    r.nblocks = err ? 0 : nb; r.chain = chain; r.stored = stored; r.fixed = fixed; r.spec = spec; r.out = out;
    if (!err) {
        const unsigned long long a = (pos + 7) >> 3;
        if (a + 4 > (unsigned long long)(im.zbits >> 3)) err = PG_E_TRUNC;                   // no Adler-32 trailer
        else if (out < (unsigned long long)im.raw) err = PG_E_SHORT;
        else {
            r.adler = (unsigned)d[a] << 24 | (unsigned)d[a + 1] << 16 | (unsigned)d[a + 2] << 8 | d[a + 3];
            r.check_adler = out == (unsigned long long)im.raw;   // more output than the image needs: libpng stops reading there
        }
    }
    r.err = err;
}

struct WordSink {
    uint32_t* w; uint32_t base; unsigned long long pos, blk, raw;
    __device__ void put(uint32_t v) { if (pos < raw) w[base + pos] = v; ++pos; }
    __device__ bool lit(uint32_t v) { put(PG_LIT | v); return true; }
    __device__ bool copy(uint32_t dd, uint32_t len) {
        if (dd > pos) return false;
        for (uint32_t k = 0; k < len; ++k) {
            if (pos >= raw) { pos += len - k; break; }
            const unsigned long long s = pos - dd;
            put(s >= blk ? w[base + s] : base + (uint32_t)s);
        }
        return true;
    }
    __device__ void stored(const uint8_t* p, uint32_t len) { for (uint32_t k = 0; k < len && pos < raw; ++k) put(PG_LIT | p[k]); }
};

// block prefix over the images (one CTA): pre[i] = blocks of images before i, pre[n] = all
__global__ void pg_block_prefix(const PgRes* __restrict__ res, int n, int* pre) {
    if (threadIdx.x) return;
    int t = 0;
    for (int i = 0; i < n; ++i) { pre[i] = t; t += res[i].err ? 0 : res[i].nblocks; }
    pre[n] = t;
}

__global__ void __launch_bounds__(PG_THREADS) pg_write(const uint8_t* __restrict__ z, const PgImg* __restrict__ imgs, int n,
                                                       const PgBlk* __restrict__ blks, const int* __restrict__ pre, uint32_t* words, PgRes* res) {
    __shared__ PmLit s_lit[PG_THREADS];
    __shared__ PmDist s_dist[PG_THREADS];
    const int total = pre[n];
    for (int g = blockIdx.x * PG_THREADS + threadIdx.x; g < total; g += gridDim.x * PG_THREADS) {
        int lo = 0, hi = n - 1;                                   // the image of block g: the last i with pre[i] <= g
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (pre[mid] <= g) lo = mid; else hi = mid - 1; }
        const PgImg& im = imgs[lo];
        const PgBlk bk = blks[im.blk0 + (g - pre[lo])];
        if (bk.out0 >= (unsigned long long)im.raw) continue;      // output past the image: libpng never reads it
        PmLit& lit = s_lit[threadIdx.x];
        PmDist& dist = s_dist[threadIdx.x];
        PmBits b;
        b.init(z + im.z0, bk.bit0, (uint64_t)im.zbits);
        b.get(1);
        const int type = (int)b.get(2);
        WordSink s{words, (uint32_t)im.w0, bk.out0, bk.out0, (unsigned long long)im.raw};
        int rc;
        if (type == PM_STORED) rc = pm_stored_body(b, s);
        else if (type == PM_FIXED) { pm_fixed_tables(lit, dist); rc = pm_huff_body(b, lit, dist, s); }
        else rc = pm_dynamic_header(b, lit, dist) ? pm_huff_body(b, lit, dist, s) : PM_BAD;
        if (rc != PM_OK) atomicOr(&res[lo].err, rc == PM_FAR ? PG_E_FAR : PG_E_DEFLATE);   // a probed block's distances are checked here
    }
}

// One round of pointer jumping over all words of the group.  flags[r] counts the words round r changed.
__global__ void __launch_bounds__(256) pg_round(uint32_t* words, long long nw, int* flags, int r) {
    if (r > 1 && ((volatile int*)flags)[r - 1] == 0) return;
    int changed = 0;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < nw; k += (long long)gridDim.x * blockDim.x) {
        const uint32_t v = words[k];
        if (v & PG_LIT) continue;
        const uint32_t s = ((volatile uint32_t*)words)[v];
        words[k] = s;
        changed = 1;
    }
    changed = __syncthreads_or(changed);
    if (threadIdx.x == 0 && changed) atomicAdd(flags + r, 1);
}

// Bytes out of the words, and per image S1 = sum of bytes, S2 = sum of (raw - k) * byte (mod 65521) for the Adler-32 check.
__global__ void __launch_bounds__(256) pg_pack(const PgImg* __restrict__ imgs, const uint32_t* __restrict__ words, uint8_t* raw, PgRes* res) {
    const PgImg& im = imgs[blockIdx.y];
    __shared__ unsigned long long sh1[8], sh2[8];
    __shared__ int sbad;
    if (threadIdx.x == 0) sbad = 0;
    __syncthreads();
    unsigned long long s1 = 0, s2 = 0;
    int bad = 0;
    if (!res[blockIdx.y].err)
        for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < im.raw; k += (long long)gridDim.x * blockDim.x) {
            const uint32_t v = words[im.w0 + k];
            bad |= !(v & PG_LIT);
            const uint32_t b = v & 0xFF;
            raw[im.w0 + k] = (uint8_t)b;
            s1 += b;
            s2 += (unsigned long long)((im.raw - k) % 65521) * b;
        }
    s1 %= 65521; s2 %= 65521;
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if ((threadIdx.x & 31) == 0) { sh1[threadIdx.x >> 5] = s1; sh2[threadIdx.x >> 5] = s2; }
    if (bad) sbad = 1;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long a = 0, c = 0;
        for (int w = 0; w < 8; ++w) { a += sh1[w]; c += sh2[w]; }
        atomicAdd(&res[blockIdx.y].s1, a % 65521);
        atomicAdd(&res[blockIdx.y].s2, c % 65521);
        if (sbad) atomicOr(&res[blockIdx.y].err, PG_E_UNRESOLVED);
    }
}

// ---------------------------------------------------------------------------------------------------------------- filters
constexpr int PG_UF_THREADS = 1024;

// One CTA per (image, pass).  Rows in bands of 1024; in a band, the thread of row r reconstructs unit x = s - r at step s (a unit is a
// pixel, or a byte below 8 bits per pixel).  Left and upper-left stay in registers, up comes from the row above's thread through
// shared memory one step later; the first row of a band reads the last row of the band before from global memory.
__global__ void __launch_bounds__(PG_UF_THREADS) pg_unfilter(const PgImg* __restrict__ imgs, uint8_t* raw, PgRes* res) {
    __shared__ uint8_t slot[2][PG_UF_THREADS][8];
    const int i = blockIdx.x / 7, ps = blockIdx.x % 7;
    const PgImg& im = imgs[i];
    if (ps >= im.npass || im.ph[ps] == 0 || res[i].err) return;
    const int bpp = im.bpp, t = threadIdx.x;
    const long long rows = im.ph[ps], rb = im.prow[ps], cols = rb / bpp;
    uint8_t* base = raw + im.w0 + im.poff[ps];
    int bad = 0;
    for (long long band = 0; band < rows; band += PG_UF_THREADS) {
        const long long r = band + t;
        const bool live = r < rows;
        uint8_t* row = base + r * (rb + 1);
        const int f = live ? row[0] : 0;
        if (f > 4) bad = 1;
        uint8_t left[8], ul[8];
        for (int j = 0; j < 8; ++j) left[j] = ul[j] = 0;
        const long long nrow = min((long long)PG_UF_THREADS, rows - band);
        const long long steps = cols + nrow - 1;
        for (long long s = 0; s < steps; ++s) {
            const long long x = s - t;
            if (live && x >= 0 && x < cols) {
                uint8_t* px = row + 1 + x * bpp;
                for (int j = 0; j < 8; ++j) {
                    if (j >= bpp) break;
                    int up = 0;
                    if (t > 0) up = slot[(s - 1) & 1][t - 1][j];
                    else if (r > 0) up = px[j - (rb + 1)];
                    const uint8_t v = pm_unfilter(f, px[j], left[j], up, ul[j]);
                    px[j] = v; left[j] = v; ul[j] = (uint8_t)up;
                    slot[s & 1][t][j] = v;
                }
            }
            __syncthreads();
        }
    }
    if (bad) atomicOr(&res[i].err, PG_E_FILTER);
}

__global__ void __launch_bounds__(256) pg_color(const PgImg* __restrict__ imgs, const uint8_t* __restrict__ raw, const uint8_t* __restrict__ pals,
                                                const PgRes* __restrict__ res, uint8_t* out) {
    const PgImg& im = imgs[blockIdx.y];
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long long)im.OW * im.OH || res[blockIdx.y].err) return;
    const int ox = (int)(pix % im.OW), oy = (int)(pix / im.OW);
    int x, y;
    jm_orient_src(im.orient, im.W, im.H, ox, oy, x, y);
    int p = 0, px = x, py = y;
    if (im.interlace) { p = pm_a7_pass(x, y); px = (x - pm_a7_x0(p)) / pm_a7_dx(p); py = (y - pm_a7_y0(p)) / pm_a7_dy(p); }
    const uint8_t* row = raw + im.w0 + im.poff[p] + (long long)py * (im.prow[p] + 1) + 1;
    const int c = im.channels, bd = im.bd;
    int R, G, B;
    if (im.ct == 3) {
        const uint8_t* e = pals + im.pal0 + 3 * pm_sample(row, px, bd, true);
        R = e[0]; G = e[1]; B = e[2];
    } else if (c <= 2) {
        R = G = B = pm_sample(row, (long long)px * c, bd, false);
    } else {
        R = pm_sample(row, (long long)px * c, bd, false); G = pm_sample(row, (long long)px * c + 1, bd, false);
        B = pm_sample(row, (long long)px * c + 2, bd, false);
    }
    uint8_t* o = out + im.out0 + pix * 3;
    o[0] = (uint8_t)B; o[1] = (uint8_t)G; o[2] = (uint8_t)R;
}

const char* pg_err_text(int e) {
    if (e & PG_E_FAR) return "invalid deflate stream (a distance reaches before the start of the data)";
    if (e & PG_E_DEFLATE) return "invalid deflate stream (bad block type, stored length, Huffman code or code lengths)";
    if (e & PG_E_TRUNC) return "the zlib stream runs past the IDAT data (truncated)";
    if (e & PG_E_SHORT) return "not enough image data";
    if (e & PG_E_ADLER) return "zlib Adler-32 mismatch (incorrect data check)";
    if (e & PG_E_FILTER) return "bad adaptive filter value (filter type above 4)";
    if (e & PG_E_BLOCKS) return "more deflate blocks than the data can hold";
    return "unresolved output byte";
}

}  // namespace

// Decodes the PNG files idx[i] of a checked call (decode.cu).  Groups of consecutive images whose transient device memory fits
// SFMB200_PNG_GROUP_BYTES run one after the other, each with one upload, one download and one host synchronisation; the images
// themselves stay on the device for the whole call.
int pg_run(sfmb200_ctx* ctx, DecodeCall& call, const std::vector<int>& idx, const std::vector<PgImage>& ims) {
    const int n = (int)idx.size();
    const bool scaled = call.scale != 1.0;
    HostPool& pool = host_pool(ctx);
    size_t zall = 0;
    for (const PgImage& p : ims) zall += p.zlen;
    if (zall >= (1ull << 29)) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "decode_images: more than 512 MB of PNG image data in one call");
    auto ow = [&](int i) { return call.ow[idx[i]]; };
    auto oh = [&](int i) { return call.oh[idx[i]]; };

    // ---- groups: consecutive images whose transient device memory fits the budget (an image alone always runs)
    auto blkcap = [&](int i) { return (long long)(ims[i].zlen * 8 / 10 + 2); };
    auto nwin = [&](int i) { return (long long)((ims[i].zlen * 8 - 16) / PG_WIN + 1); };
    auto transient = [&](int i) {
        return al256(ims[i].zlen + 16) + al256(sizeof(PgCand) * PG_CAP * nwin(i)) + al256(5ull * ims[i].raw) + al256(8ull * blkcap(i)) + al256(sizeof(PgImg) + 768 + sizeof(PgRes))
             + (scaled ? al256((size_t)ims[i].OW * ims[i].OH * 3) : 0);
    };
    std::vector<int> g0{0};
    size_t acc = 0;
    for (int i = 0; i < n; ++i) {
        const size_t t = transient(i);
        if (i > g0.back() && acc + t > (size_t)SFMB200_PNG_GROUP_BYTES) { g0.push_back(i); acc = 0; }
        acc += t;
    }
    g0.push_back(n);
    const int ngroups = (int)g0.size() - 1;
    // the images, in caller order, each behind its group's result words: one contiguous download per group
    std::vector<size_t> img_off(n), grp_off(ngroups + 1);
    size_t a = 0;
    for (int g = 0; g < ngroups; ++g) {
        grp_off[g] = a;
        a += al256(sizeof(PgRes) * (g0[g + 1] - g0[g]) + sizeof(int) * (PG_ROUNDS + 1));
        for (int i = g0[g]; i < g0[g + 1]; ++i) {
            img_off[i] = a; a += al256((size_t)ow(i) * oh(i) * 3);
        }
    }
    grp_off[ngroups] = a;
    const size_t keep_bytes = a;
    size_t trans_max = 0;
    for (int g = 0; g < ngroups; ++g) {
        size_t t = 0;
        for (int i = g0[g]; i < g0[g + 1]; ++i) t += transient(i);
        trans_max = std::max(trans_max, t);
    }
    // one reservation for the call (the images must not move between groups); the resize descriptors and taps of a group are small
    SFM_CUDA(ctx, ctx->png_dev.reserve(al256(keep_bytes) + trans_max + (4u << 20)));
    char* keep = (char*)ctx->png_dev.p;
    char* dv = keep + al256(keep_bytes);
    cudaStream_t st = ctx->stream;
    int64_t up_total = 0, down_total = 0, rounds = 0, blocks = 0, chain = 0, stored = 0, fixed = 0, spec = 0, probed = 0;

    for (int g = 0; g < ngroups; ++g) {
        const int a0 = g0[g], m = g0[g + 1] - a0;
        // ---- group layout
        std::vector<PgImg> img(m);
        std::vector<RzImg> grz;
        std::vector<RzTap> taps;
        size_t zbytes = 0;
        long long words = 0, blks = 0, full = 0, wins = 0;
        for (int k = 0; k < m; ++k) {
            const PgImage& p = ims[a0 + k];
            PgImg& d = img[k];
            memset(&d, 0, sizeof d);
            d.z0 = (long long)zbytes; d.zbits = (long long)p.zlen * 8; zbytes += al256(p.zlen + 16);
            d.w0 = words; d.raw = p.raw; words += (p.raw + 15) & ~15ll;
            d.blk0 = blks; d.blkcap = blkcap(a0 + k); blks += d.blkcap;
            d.pal0 = 768ll * k;
            d.win0 = wins; d.nwin = nwin(a0 + k); wins += d.nwin;
            d.W = p.W; d.H = p.H; d.OW = p.OW; d.OH = p.OH; d.orient = p.orient; d.bd = p.bd; d.ct = p.ct; d.channels = p.channels;
            d.bpp = p.bpp; d.npass = p.npass; d.interlace = p.interlace;
            for (int q = 0; q < 7; ++q) { d.pw[q] = p.pw[q]; d.ph[q] = p.ph[q]; d.prow[q] = p.prow[q]; d.poff[q] = p.poff[q]; }
            if (scaled) { d.out0 = full; full += (long long)al256((size_t)p.OW * p.OH * 3); }
            else d.out0 = (long long)(img_off[a0 + k] - grp_off[g]);
        }
        if (words >= (1ll << 31)) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "image %d: too much image data for one group", idx[a0]);
        if (scaled) {
            grz.resize(m);
            for (int k = 0; k < m; ++k) { memset(&grz[k], 0, sizeof(RzImg)); grz[k].sw = img[k].OW; grz[k].sh = img[k].OH; }
            rz_plan(call.scale, grz.data(), m, taps, nullptr);
            for (int k = 0; k < m; ++k) {
                grz[k].src0 = img[k].out0; grz[k].src_stride = (long long)img[k].OW * 3;
                grz[k].dst0 = (long long)(img_off[a0 + k] - grp_off[g]); grz[k].dst_stride = (long long)grz[k].dw * 3;
            }
        }
        const size_t o_img = 0, o_pal = o_img + al256(sizeof(PgImg) * m), o_rz = o_pal + al256(768ull * m);
        const size_t o_tap = o_rz + al256(sizeof(RzImg) * grz.size()), o_z = o_tap + al256(sizeof(RzTap) * taps.size());
        const size_t up_bytes = o_z + zbytes;
        SFM_CUDA(ctx, ctx->png_pin_up.reserve(up_bytes));
        char* up = (char*)ctx->png_pin_up.p;
        memcpy(up + o_img, img.data(), sizeof(PgImg) * m);
        if (scaled) { memcpy(up + o_rz, grz.data(), sizeof(RzImg) * m); memcpy(up + o_tap, taps.data(), sizeof(RzTap) * taps.size()); }
        pool.parallel_for(m, [&](int k) {
            const PgImage& p = ims[a0 + k];
            memcpy(up + o_pal + 768ull * k, p.pal, 768);
            char* zd = up + o_z + img[k].z0;
            size_t o = 0;
            for (auto& c : p.idat) { memcpy(zd + o, call.data[idx[a0 + k]] + c.first, c.second); o += c.second; }
            memset(zd + o, 0, al256(p.zlen + 16) - o);
        });
        // ---- device memory of the group
        const size_t d_words = al256(up_bytes), d_raw = d_words + al256(4ull * words), d_blk = d_raw + al256((size_t)words + 16);
        const size_t d_pre = d_blk + al256(sizeof(PgBlk) * blks), d_cand = d_pre + al256(sizeof(int) * (m + 1));
        const size_t d_full = d_cand + al256(sizeof(PgCand) * PG_CAP * wins);
        const size_t total = d_full + (size_t)full;
        if (al256(keep_bytes) + total > ctx->png_dev.cap)
            return sfmb200_fail(ctx, SFMB200_ERR_NOMEM, "decode_images: group %d needs %zu bytes past the images", g, total);
        char* down = keep + grp_off[g];
        PgRes* d_res = (PgRes*)down;
        int* d_flags = (int*)(down + sizeof(PgRes) * m);
        const size_t res_bytes = sizeof(PgRes) * m + sizeof(int) * (PG_ROUNDS + 1);
        uint8_t* d_out = (uint8_t*)down;                   // image offsets (out0, dst0) are relative to the group's download
        const PgImg* d_img = (const PgImg*)(dv + o_img);
        const uint8_t* d_pal = (const uint8_t*)(dv + o_pal);
        const uint8_t* d_z = (const uint8_t*)(dv + o_z);
        uint32_t* d_w = (uint32_t*)(dv + d_words);
        uint8_t* d_r = (uint8_t*)(dv + d_raw);
        PgBlk* d_b = (PgBlk*)(dv + d_blk);
        int* d_p = (int*)(dv + d_pre);
        PgCand* d_c = (PgCand*)(dv + d_cand);
        uint8_t* d_f = scaled ? (uint8_t*)(dv + d_full) : d_out;
        SFM_CUDA(ctx, cudaMemcpyAsync(dv, up, up_bytes, cudaMemcpyHostToDevice, st));
        SFM_CUDA(ctx, cudaMemsetAsync(down, 0, res_bytes, st));
        // every word starts resolved: the padding between images (and an image whose chain failed) is never written, and pg_round
        // sweeps the whole array
        SFM_CUDA(ctx, cudaMemsetAsync(d_w, 0xFF, 4ull * words, st));
        SFM_CUDA(ctx, cudaMemsetAsync(d_c, 0xFF, sizeof(PgCand) * PG_CAP * wins, st));
        const int sg = (int)std::min<long long>(ceil_div64(wins, PG_THREADS), (long long)ctx->sm_count * 64);
        pg_scan<<<sg, PG_THREADS, 0, st>>>(d_z, d_img, m, wins, d_c);
        SFM_LAUNCH_CHECK(ctx);
        pg_probe<<<ctx->sm_count * 8, PG_THREADS, 0, st>>>(d_z, d_img, m, wins * PG_CAP, d_c, d_res);
        SFM_LAUNCH_CHECK(ctx);
        pg_chain<<<ceil_div(m, PG_THREADS), PG_THREADS, 0, st>>>(d_z, d_img, m, d_c, d_b, d_res);
        SFM_LAUNCH_CHECK(ctx);
        pg_block_prefix<<<1, 32, 0, st>>>(d_res, m, d_p);
        SFM_LAUNCH_CHECK(ctx);
        pg_write<<<ctx->sm_count * 8, PG_THREADS, 0, st>>>(d_z, d_img, m, d_b, d_p, d_w, d_res);
        SFM_LAUNCH_CHECK(ctx);
        const int rb = (int)std::min<long long>(ceil_div64(words, 256), (long long)ctx->sm_count * 16);
        for (int r = 1; r <= PG_ROUNDS; ++r) {
            pg_round<<<std::max(rb, 1), 256, 0, st>>>(d_w, words, d_flags, r);
            SFM_LAUNCH_CHECK(ctx);
        }
        long long max_raw = 0, max_pix = 0;
        for (auto& d : img) { max_raw = std::max(max_raw, d.raw); max_pix = std::max(max_pix, (long long)d.OW * d.OH); }
        pg_pack<<<dim3((unsigned)std::min<long long>(ceil_div64(max_raw, 256 * 16), 1024), (unsigned)m), 256, 0, st>>>(d_img, d_w, d_r, d_res);
        SFM_LAUNCH_CHECK(ctx);
        pg_unfilter<<<7 * m, PG_UF_THREADS, 0, st>>>(d_img, d_r, d_res);
        SFM_LAUNCH_CHECK(ctx);
        pg_color<<<dim3((unsigned)ceil_div64(max_pix, 256), (unsigned)m), 256, 0, st>>>(d_img, d_r, d_pal, d_res, d_f);
        SFM_LAUNCH_CHECK(ctx);
        if (scaled)
            if (int rc = rz_enqueue(ctx, call.scale, grz.data(), m, (const RzImg*)(dv + o_rz), (const RzTap*)(dv + o_tap), d_f, d_out)) return rc;
        const size_t got = call.out_bgr ? grp_off[g + 1] - grp_off[g] : res_bytes;
        SFM_CUDA(ctx, ctx->png_pin_down.reserve(got));
        char* hd = (char*)ctx->png_pin_down.p;
        SFM_CUDA(ctx, cudaMemcpyAsync(hd, down, got, cudaMemcpyDeviceToHost, st));
        SFM_CUDA(ctx, cudaStreamSynchronize(st));
        up_total += (int64_t)up_bytes; down_total += (int64_t)got;
        const PgRes* hr = (const PgRes*)hd;
        const int* hf = (const int*)(hd + sizeof(PgRes) * m);
        int r = 1;
        while (r <= PG_ROUNDS && hf[r]) ++r;
        rounds += r;
        for (int k = 0; k < m; ++k) {
            int e = hr[k].err;
            if (!e && hr[k].check_adler) {
                const unsigned A = (unsigned)((1 + hr[k].s1) % 65521), B = (unsigned)(((unsigned long long)img[k].raw % 65521 + hr[k].s2) % 65521);
                if ((B << 16 | A) != hr[k].adler) e = PG_E_ADLER;
            }
            if (e) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: %s", idx[a0 + k], pg_err_text(e));
            blocks += hr[k].nblocks; chain += hr[k].chain; stored += hr[k].stored; fixed += hr[k].fixed; spec += hr[k].spec;
            probed += hr[k].probed;
        }
        if (call.out_bgr)
            pool.parallel_for(m, [&](int k) {
                const int i = a0 + k, j = idx[i];
                const size_t row = (size_t)ow(i) * 3;
                copy_rows(call.out_bgr[j], call.stride(j), (const uint8_t*)(hd + (img_off[i] - grp_off[g])), row, row, oh(i));
            });
    }
    int64_t* s = ctx->png_stats;
    s[0] = blocks; s[1] = spec; s[2] = chain; s[3] = probed; s[4] = rounds; s[5] = up_total; s[6] = down_total; s[7] = ngroups; s[8] = stored; s[9] = fixed;
    for (int i = 0; i < n; ++i) call.dev[idx[i]] = (const uint8_t*)(keep + img_off[i]);
    return SFMB200_OK;
}

extern "C" {

int sfmb200_png_last_stats(const sfmb200_ctx* ctx, int64_t* stats) {
    if (!ctx || !stats) return SFMB200_ERR_INVALID;
    for (int k = 0; k < SFMB200_PNG_STATS; ++k) stats[k] = ctx->png_stats[k];
    return SFMB200_OK;
}

}  // extern "C"
