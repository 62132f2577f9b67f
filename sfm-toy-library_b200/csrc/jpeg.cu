// jpeg.cu -- JPEG decoding of a batch of files on the device, byte-identical to cv::imread(IMREAD_COLOR) (include/sfmb200.h).
//
// The host parses the markers (jpeg_parse.h) and packs the tables, the layout and the entropy-coded bytes of every image into one
// pinned buffer: one upload.  On the device:
//   jd_unstuff        removes the FF00 stuffing and the RSTn markers, one 4 KB chunk per CTA (block prefix sum of kept bytes)
//   jd_sync0          every subsequence of JD_SUB bits decoded from a guessed state (block 0 of the MCU, DC)
//   jd_sync_round     up to JD_ROUNDS rounds: a subsequence whose predecessor's exit moved is decoded again from that exit
//   jd_sync_sweep     one warp per segment finishes the fixed point in order (rarely has anything left to do)
//   scan of blocks    first block of every subsequence (prefix sum of the block counts)
//   jd_write          decodes every subsequence once more from its true entry and writes int16[64] coefficient blocks
//   jd_dc_sum + scan + jd_dc_apply   DC prediction: per-component prefix sums over MCUs, reset at every restart segment
//   jd_idct           dequantisation and jpeg_idct_islow, 8 threads per block, into uint8 component planes
//   jd_color          upsampling, YCbCr -> B,G,R and the EXIF orientation, into the download area
//   rz_*              (sfmb200_decode_jpeg_batch_scaled only) jd_color writes to device memory and the downscale of resize.cu
//                     writes the resized images into the download area instead
// then one download (per-image error flags, statistics and the images) and one host synchronisation.
#include "common.cuh"
#include "jpeg_parse.h"
#include "resize_math.cuh"

namespace {

constexpr int JD_CHUNK = 4096;        // bytes per unstuffing CTA
constexpr uint32_t JD_SUB = 1024;     // bits per subsequence
constexpr int JD_ROUNDS = 6;          // parallel synchronisation rounds before the in-order sweep
constexpr int JD_ERR_DATA = 1, JD_ERR_SHORT = 2;

struct JdImg {
    int W, H, OW, OH, orient, ncomp, mcus_x, restart;
    int hs[3], vs[3], hr[3], vr[3], cw[3], ch[3], wb[3], hb[3];
    long long blk0[3], plane0[3], out0, mcu0, nmcu, nblocks;
    JmScan scan;
    int tab0;                          // first of the image's 8 Huffman tables
};
struct JdSeg { uint32_t b0, b1; int img, first_sub, nsub, n_mcu; long long first_mcu; };
struct JdChunk { uint32_t in0, len, out0, flags; };   // flags: 1 = first chunk of an image's scan, 2 = last
struct JdStats { unsigned long long cw_first, cw_extra, rounds, swept; };

__device__ __forceinline__ bool is_rst(uint32_t b) { return b >= 0xD0 && b <= 0xD7; }

// ---------------------------------------------------------------------------------------------------------------- unstuffing
__global__ void __launch_bounds__(256) jd_unstuff(const uint8_t* __restrict__ in, const JdChunk* __restrict__ chunks, uint8_t* __restrict__ out) {
    const JdChunk c = chunks[blockIdx.x];
    __shared__ int warp_sum[8];
    const int t = threadIdx.x, i0 = t * 16;
    uint32_t keep = 0;
    int cnt = 0;
    for (int q = 0; q < 16; ++q) {
        const int i = i0 + q;
        if (i >= (int)c.len) break;
        const uint32_t g = c.in0 + i;
        const uint32_t b = in[g];
        const uint32_t prev = (i > 0 || !(c.flags & 1)) ? in[g - 1] : 0;
        const uint32_t next = (i + 1 < (int)c.len || !(c.flags & 2)) ? in[g + 1] : 0;
        const bool drop = (prev == 0xFF && (b == 0 || is_rst(b))) || (b == 0xFF && is_rst(next));
        if (!drop) { keep |= 1u << q; ++cnt; }
    }
    int incl = cnt;
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if ((t & 31) >= o) incl += v; }
    if ((t & 31) == 31) warp_sum[t >> 5] = incl;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < (t >> 5); ++w) base += warp_sum[w];
    uint32_t o = c.out0 + base + incl - cnt;
    for (int q = 0; q < 16; ++q)
        if (keep >> q & 1) out[o++] = in[c.in0 + i0 + q];
}

// ---------------------------------------------------------------------------------------------------------------- Huffman
__device__ __forceinline__ uint32_t sub_start(const JdSeg& s, int j) { return s.b0 + (uint32_t)(j - s.first_sub) * JD_SUB; }
__device__ __forceinline__ uint32_t sub_stop(const JdSeg& s, int j) { return j + 1 == s.first_sub + s.nsub ? s.b1 : sub_start(s, j + 1); }

__device__ __forceinline__ void count_codewords(unsigned long long* ctr, int cw) {
    for (int o = 16; o > 0; o >>= 1) cw += __shfl_xor_sync(0xffffffffu, cw, o);
    if ((threadIdx.x & 31) == 0 && cw) atomicAdd(ctr, (unsigned long long)cw);
}

__global__ void __launch_bounds__(128) jd_sync0(const uint8_t* __restrict__ u, const JdSeg* __restrict__ segs, const int* __restrict__ sub_seg,
                                                const JdImg* __restrict__ imgs, const JmHuff* __restrict__ tabs, int nsub, uint64_t* exits,
                                                int* computed, int* changed, JdStats* st) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    int cw = 0;
    if (j < nsub) {
        const JdSeg s = segs[sub_seg[j]];
        const JdImg& im = imgs[s.img];
        JmNoSink none;
        exits[j] = jm_span(u, sub_start(s, j), 0, sub_stop(s, j), s.b1, im.scan, tabs + im.tab0, none, &cw);
        computed[j] = 0; changed[j] = 0;
    }
    count_codewords(&st->cw_first, cw);
}

__global__ void __launch_bounds__(128) jd_sync_round(const uint8_t* __restrict__ u, const JdSeg* __restrict__ segs, const int* __restrict__ sub_seg,
                                                     const JdImg* __restrict__ imgs, const JmHuff* __restrict__ tabs, int nsub, uint64_t* exits,
                                                     int* computed, int* changed, int* round_changes, int r, JdStats* st) {
    if (r > 1 && ((volatile int*)round_changes)[r - 1] == 0) return;        // the previous round moved nothing: converged
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    int cw = 0;
    if (j < nsub) {
        const JdSeg s = segs[sub_seg[j]];
        if (j != s.first_sub && ((volatile int*)changed)[j - 1] >= computed[j]) {
            const JdImg& im = imgs[s.img];
            JmNoSink none;
            const uint64_t entry = ((volatile uint64_t*)exits)[j - 1];
            const uint64_t e = jm_span(u, jm_exit_pos(entry), jm_exit_state(entry), sub_stop(s, j), s.b1, im.scan, tabs + im.tab0, none, &cw);
            computed[j] = r;
            if (!jm_exit_same(e, exits[j])) { ((volatile int*)changed)[j] = r; atomicAdd(round_changes + r, 1); }
            ((volatile uint64_t*)exits)[j] = e;
        }
    }
    if (threadIdx.x == 0 && blockIdx.x == 0) atomicMax(&st->rounds, (unsigned long long)r);
    count_codewords(&st->cw_extra, cw);
}

// One warp per segment: in order, every subsequence whose predecessor's exit moved after it was last decoded is decoded again.
__global__ void __launch_bounds__(128) jd_sync_sweep(const uint8_t* __restrict__ u, const JdSeg* __restrict__ segs, int nseg,
                                                     const JdImg* __restrict__ imgs, const JmHuff* __restrict__ tabs, uint64_t* exits,
                                                     int* computed, int* changed, const int* round_changes, JdStats* st) {
    if (round_changes[JD_ROUNDS] == 0) return;
    const int sidx = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (sidx >= nseg) return;
    const JdSeg s = segs[sidx];
    const JdImg& im = imgs[s.img];
    int cw = 0, swept = 0;
    for (int j0 = s.first_sub + 1; j0 < s.first_sub + s.nsub;) {
        const int j = j0 + lane;
        const bool need = j < s.first_sub + s.nsub && changed[j - 1] >= computed[j];
        const unsigned m = __ballot_sync(0xffffffffu, need);
        if (!m) { j0 += 32; continue; }
        const int jj = j0 + __ffs(m) - 1;
        if (lane == 0) {
            JmNoSink none;
            const uint64_t entry = exits[jj - 1];
            const uint64_t e = jm_span(u, jm_exit_pos(entry), jm_exit_state(entry), sub_stop(s, jj), s.b1, im.scan, tabs + im.tab0, none, &cw);
            computed[jj] = JD_ROUNDS + 1;
            if (!jm_exit_same(e, exits[jj])) changed[jj] = JD_ROUNDS + 1;
            exits[jj] = e;
            ++swept;
        }
        __syncwarp();
        j0 = jj + 1;
    }
    if (lane == 0 && swept) {
        atomicAdd(&st->cw_extra, (unsigned long long)cw);
        atomicAdd(&st->swept, (unsigned long long)swept);
    }
}

__global__ void jd_nblk(const uint64_t* __restrict__ exits, int nsub, uint32_t* nblk) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < nsub) nblk[j] = (uint32_t)jm_exit_nblk(exits[j]);
}

// coefficient block of block b of the image's MCU number mcu
__device__ __forceinline__ int16_t* block_ptr(int16_t* coef, const JdImg& im, long long mcu, int b) {
    const int c = im.scan.blk_comp[b];
    const long long bx = (mcu % im.mcus_x) * im.hs[c] + im.scan.blk_dx[b], by = (mcu / im.mcus_x) * im.vs[c] + im.scan.blk_dy[b];
    return coef + 64 * (im.blk0[c] + by * im.wb[c] + bx);
}

struct WriteSink {
    int16_t* blocks; const JdImg* im; long long first_mcu, base, expected; int* err;
    long long cur = -(1ll << 40); int16_t* ptr = nullptr;
    __device__ void coef_at(long long o, int k, int v) {
        if (o != cur) { cur = o; ptr = block_ptr(blocks, *im, first_mcu + o / im->scan.bpm, (int)(o % im->scan.bpm)); }
        ptr[jm_natural(k)] = (int16_t)v;
    }
    __device__ void coef(int ord, int k, int v) {
        const long long o = base + ord;
        if (o < 0) { *err |= JD_ERR_DATA; return; }
        if (o < expected) coef_at(o, k, v);
    }
    __device__ void fail(int ord, int) { if (base + ord < expected) *err |= JD_ERR_DATA; }
};

__global__ void __launch_bounds__(128) jd_write(const uint8_t* __restrict__ u, const JdSeg* __restrict__ segs, const int* __restrict__ sub_seg,
                                                const JdImg* __restrict__ imgs, const JmHuff* __restrict__ tabs, int nsub, const uint64_t* __restrict__ exits,
                                                const uint32_t* __restrict__ blkpre, int16_t* coef, int* img_err) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nsub) return;
    const JdSeg s = segs[sub_seg[j]];
    const JdImg& im = imgs[s.img];
    int err = 0;
    WriteSink sink{coef, &im, s.first_mcu, (long long)(blkpre[j] - blkpre[s.first_sub]), (long long)s.n_mcu * im.scan.bpm, &err};
    const uint64_t entry = j == s.first_sub ? jm_pack_exit(s.b0, 0, 0) : exits[j - 1];
    jm_span(u, jm_exit_pos(entry), jm_exit_state(entry), sub_stop(s, j), s.b1, im.scan, tabs + im.tab0, sink);
    if (j + 1 == s.first_sub + s.nsub && sink.base + jm_exit_nblk(exits[j]) < sink.expected) err |= JD_ERR_SHORT;
    if (err) atomicOr(img_err + s.img, err);
}

// ---------------------------------------------------------------------------------------------------------------- scans
struct AddU32 {
    typedef uint32_t T;
    __device__ static T id() { return 0; }
    __device__ static T op(T a, T b) { return a + b; }
};
struct Add3x16 {                       // three DC predictors of an MCU, each modulo 2^16 (the int16 truncation libjpeg ends with)
    typedef unsigned long long T;
    __device__ static T id() { return 0; }
    __device__ static T op(T a, T b) {
        T r = 0;
        for (int l = 0; l < 3; ++l) r |= (((a >> (16 * l)) + (b >> (16 * l))) & 0xffffull) << (16 * l);
        return r;
    }
};

constexpr int SCAN_ITEMS = 4, SCAN_THREADS = 256, SCAN_TILE = SCAN_ITEMS * SCAN_THREADS;

template <class Op>
__device__ typename Op::T block_excl_scan(typename Op::T v, typename Op::T& total) {
    typedef typename Op::T T;
    __shared__ T ws[SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    T incl = v;
    for (int o = 1; o < 32; o <<= 1) { const T x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl = Op::op(x, incl); }
    if (lane == 31) ws[w] = incl;
    __syncthreads();
    T base = Op::id(), tot = Op::id();
    for (int k = 0; k < SCAN_THREADS / 32; ++k) { if (k < w) base = Op::op(base, ws[k]); tot = Op::op(tot, ws[k]); }
    __syncthreads();
    total = tot;
    const T ex = __shfl_up_sync(0xffffffffu, incl, 1);
    return Op::op(base, lane ? ex : Op::id());
}

template <class Op>
__global__ void __launch_bounds__(SCAN_THREADS) scan_reduce(const typename Op::T* in, long long n, typename Op::T* part) {
    typedef typename Op::T T;
    T s = Op::id();
    const long long i0 = (long long)blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    for (int q = 0; q < SCAN_ITEMS; ++q) if (i0 + q < n) s = Op::op(s, in[i0 + q]);
    T total;
    block_excl_scan<Op>(s, total);
    if (threadIdx.x == 0) part[blockIdx.x] = total;
}

template <class Op>
__global__ void __launch_bounds__(SCAN_THREADS) scan_parts(typename Op::T* part, int np) {
    typedef typename Op::T T;
    T carry = Op::id();
    for (int t0 = 0; t0 < np; t0 += SCAN_THREADS) {
        const int i = t0 + threadIdx.x;
        const T v = i < np ? part[i] : Op::id();
        T total;
        const T ex = block_excl_scan<Op>(v, total);
        if (i < np) part[i] = Op::op(carry, ex);
        carry = Op::op(carry, total);
    }
}

template <class Op>
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply(const typename Op::T* in, long long n, const typename Op::T* part, typename Op::T* out) {
    typedef typename Op::T T;
    const long long i0 = (long long)blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    T v[SCAN_ITEMS], s = Op::id();
    for (int q = 0; q < SCAN_ITEMS; ++q) { v[q] = i0 + q < n ? in[i0 + q] : Op::id(); s = Op::op(s, v[q]); }
    T total;
    T run = Op::op(part[blockIdx.x], block_excl_scan<Op>(s, total));
    for (int q = 0; q < SCAN_ITEMS; ++q) { if (i0 + q < n) out[i0 + q] = run; run = Op::op(run, v[q]); }
}

template <class Op>
int excl_scan(sfmb200_ctx* ctx, const typename Op::T* in, long long n, typename Op::T* part, typename Op::T* out) {
    if (n <= 0) return SFMB200_OK;
    const int nb = (int)ceil_div64(n, SCAN_TILE);
    scan_reduce<Op><<<nb, SCAN_THREADS, 0, ctx->stream>>>(in, n, part);
    SFM_LAUNCH_CHECK(ctx);
    scan_parts<Op><<<1, SCAN_THREADS, 0, ctx->stream>>>(part, nb);
    SFM_LAUNCH_CHECK(ctx);
    scan_apply<Op><<<nb, SCAN_THREADS, 0, ctx->stream>>>(in, n, part, out);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

// ---------------------------------------------------------------------------------------------------------------- DC prediction
__global__ void jd_dc_sum(const JdImg* __restrict__ imgs, const int16_t* __restrict__ coef, unsigned long long* mcu_sum) {
    const JdImg& im = imgs[blockIdx.y];
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= im.nmcu) return;
    unsigned long long r = 0;
    for (int b = 0; b < im.scan.bpm; ++b) {
        const uint16_t d = (uint16_t)block_ptr((int16_t*)coef, im, m, b)[0];
        r = Add3x16::op(r, (unsigned long long)d << (16 * im.scan.blk_comp[b]));
    }
    mcu_sum[im.mcu0 + m] = r;
}

__global__ void jd_dc_apply(const JdImg* __restrict__ imgs, int16_t* coef, const unsigned long long* __restrict__ mcu_pre) {
    const JdImg& im = imgs[blockIdx.y];
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= im.nmcu) return;
    const long long f = im.restart ? m / im.restart * im.restart : 0;     // first MCU of the restart segment
    const unsigned long long a = mcu_pre[im.mcu0 + m], z = mcu_pre[im.mcu0 + f];
    unsigned long long run = 0;
    for (int l = 0; l < 3; ++l) run |= (((a >> (16 * l)) - (z >> (16 * l))) & 0xffffull) << (16 * l);
    for (int b = 0; b < im.scan.bpm; ++b) {
        int16_t* p = block_ptr(coef, im, m, b);
        const int c = im.scan.blk_comp[b];
        run = Add3x16::op(run, (unsigned long long)(uint16_t)p[0] << (16 * c));
        p[0] = (int16_t)(uint16_t)(run >> (16 * c));
    }
}

// ---------------------------------------------------------------------------------------------------------------- IDCT, colour
__global__ void __launch_bounds__(256) jd_idct(const JdImg* __restrict__ imgs, const int16_t* __restrict__ coef, const int16_t* __restrict__ qt,
                                               uint8_t* planes) {
    __shared__ int ws[32][64];
    const JdImg& im = imgs[blockIdx.y];
    const long long ib = (long long)blockIdx.x * 32 + threadIdx.x / 8;
    const int t = threadIdx.x & 7, slot = threadIdx.x / 8;
    const bool live = ib < im.nblocks;
    int c = 0;
    while (live && c + 1 < im.ncomp && im.blk0[0] + ib >= im.blk0[c + 1]) ++c;
    const long long lb = im.blk0[0] + ib - im.blk0[c];
    const int16_t* blk = coef + 64 * (im.blk0[0] + ib);
    const int16_t* q = qt + 64 * (3 * blockIdx.y + c);
    if (live) jm_idct_col(blk, q, t, ws[slot]);
    __syncwarp();
    if (!live) return;
    uint8_t row[8];
    jm_idct_row(ws[slot], t, row);
    const long long bx = lb % im.wb[c], by = lb / im.wb[c];
    const long long stride = (long long)im.wb[c] * 8;
    uint2 v;
    v.x = row[0] | row[1] << 8 | row[2] << 16 | (uint32_t)row[3] << 24;
    v.y = row[4] | row[5] << 8 | row[6] << 16 | (uint32_t)row[7] << 24;
    *(uint2*)(planes + im.plane0[c] + (by * 8 + t) * stride + bx * 8) = v;
}

__global__ void __launch_bounds__(256) jd_color(const JdImg* __restrict__ imgs, const uint8_t* __restrict__ planes, uint8_t* out) {
    const JdImg& im = imgs[blockIdx.y];
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long long)im.OW * im.OH) return;
    const int ox = (int)(pix % im.OW), oy = (int)(pix / im.OW);
    int x, y;
    jm_orient_src(im.orient, im.W, im.H, ox, oy, x, y);
    uint8_t* o = out + im.out0 + pix * 3;
    const int Y = planes[im.plane0[0] + (long long)y * im.wb[0] * 8 + x];
    if (im.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; return; }
    const int cb = jm_chroma(planes + im.plane0[1], im.wb[1] * 8, im.cw[1], im.ch[1], im.hr[1], im.vr[1], x, y);
    const int cr = jm_chroma(planes + im.plane0[2], im.wb[2] * 8, im.cw[2], im.ch[2], im.hr[2], im.vr[2], x, y);
    uint8_t bgr[3];
    jm_ycc_to_bgr(Y, cb, cr, bgr);
    o[0] = bgr[0]; o[1] = bgr[1]; o[2] = bgr[2];
}

size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

}  // namespace

// Both decode entry points.  scale == 1: jd_color writes the images into the download area.  Otherwise jd_color writes them to device
// memory, resize.cu's kernels downscale them into the download area, and only the resized images come back.
static int jd_decode(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, uint8_t* const* out_bgr,
                     const size_t* out_stride) {
    if (!ctx) return SFMB200_ERR_INVALID;
    if (n < 0 || (n > 0 && (!data || !size || !out_bgr))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "decode_jpeg_batch: bad arguments");
    if (n > 65535) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "decode_jpeg_batch: at most 65535 images per call");
    if (!std::isfinite(scale) || scale <= 0)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "decode_jpeg_batch_scaled: scale %g is not a positive finite number", scale);
    const bool scaled = scale != 1.0;
    for (int i = 0; i < 7; ++i) ctx->jpeg_stats[i] = 0;
    if (n == 0) return SFMB200_OK;
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->pool) ctx->pool = new HostPool(HostPool::default_threads() - 1);
    HostPool& pool = *ctx->pool;

    // ---- parse every file (host threads)
    std::vector<JpImage> ims(n);
    std::vector<int> rcs(n, 0);
    std::vector<std::string> whys(n);
    pool.parallel_for(n, [&](int i) { rcs[i] = jp_parse(data[i], size[i], JD_CHUNK, ims[i], whys[i]); });
    for (int i = 0; i < n; ++i) {
        if (rcs[i]) return sfmb200_fail(ctx, rcs[i], "image %d: %s", i, whys[i].c_str());
        if (!out_bgr[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: no output buffer", i);
    }
    // ---- the downscale: output sizes and taps of every image
    std::vector<RzImg> rz(scaled ? n : 0);
    std::vector<RzTap> taps;
    if (scaled) {
        for (int i = 0; i < n; ++i) { memset(&rz[i], 0, sizeof(RzImg)); rz[i].sw = ims[i].OW; rz[i].sh = ims[i].OH; }
        int bad = 0;
        if (!rz_plan(scale, rz.data(), n, taps, &bad))
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: scale %g of a %dx%d image gives no image", bad, scale, ims[bad].OW, ims[bad].OH);
    }
    for (int i = 0; i < n; ++i) {
        const int ow = scaled ? rz[i].dw : ims[i].OW;
        if (out_stride && out_stride[i] && out_stride[i] < (size_t)ow * 3)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: output stride %zu < %d", i, out_stride[i], ow * 3);
    }

    // ---- layout
    std::vector<JdImg> img(n);
    std::vector<JdSeg> segs;
    std::vector<JdChunk> chunks;
    std::vector<size_t> in0(n);
    size_t in_bytes = 0, ubytes = 0;
    long long blocks = 0, mcus = 0, planes = 0, outb = 0, rzb = 0;    // outb: decoded images; rzb: resized images
    for (int i = 0; i < n; ++i) {
        const JpImage& p = ims[i];
        JdImg& d = img[i];
        memset(&d, 0, sizeof d);
        d.W = p.W; d.H = p.H; d.OW = p.OW; d.OH = p.OH; d.orient = p.orient; d.ncomp = p.ncomp; d.mcus_x = p.mcus_x; d.restart = p.restart;
        for (int c = 0; c < p.ncomp; ++c) {
            d.hs[c] = p.hs[c]; d.vs[c] = p.vs[c]; d.hr[c] = p.hmax / p.hs[c]; d.vr[c] = p.vmax / p.vs[c];
            d.cw[c] = p.cw[c]; d.ch[c] = p.ch[c]; d.wb[c] = p.wb[c]; d.hb[c] = p.hb[c];
            d.blk0[c] = blocks; blocks += (long long)p.wb[c] * p.hb[c];
            d.plane0[c] = planes; planes += (long long)al256((size_t)p.wb[c] * p.hb[c] * 64);
        }
        d.nblocks = blocks - d.blk0[0];
        d.out0 = outb; outb += (long long)al256((size_t)p.OW * p.OH * 3);
        if (scaled) {
            RzImg& r = rz[i];
            r.src0 = d.out0; r.src_stride = (long long)p.OW * 3;
            r.dst0 = rzb; r.dst_stride = (long long)r.dw * 3; rzb += (long long)al256((size_t)r.dst_stride * r.dh);
        }
        d.mcu0 = mcus; d.nmcu = p.mcus(); mcus += d.nmcu;
        d.scan = p.scan; d.tab0 = 8 * i;
        // chunks of the scan (aligned, so that every chunk belongs to one image) and the unstuffed positions
        in0[i] = in_bytes;
        const size_t nch = p.seg_skip.size();
        size_t u = ubytes;
        for (size_t k = 0; k < nch; ++k) {
            JdChunk ch;
            ch.in0 = (uint32_t)(in_bytes + k * JD_CHUNK);
            ch.len = (uint32_t)std::min<size_t>(JD_CHUNK, p.scan_len - k * JD_CHUNK);
            ch.out0 = (uint32_t)u;
            ch.flags = (k == 0 ? 1u : 0u) | (k + 1 == nch ? 2u : 0u);
            u += ch.len - p.seg_skip[k];
            chunks.push_back(ch);
        }
        in_bytes += nch * JD_CHUNK;
        const long long R = p.restart ? p.restart : d.nmcu;
        for (size_t k = 0; k < p.seg_bytes.size(); ++k) {
            JdSeg s;
            s.b0 = (uint32_t)(ubytes * 8); ubytes += p.seg_bytes[k]; s.b1 = (uint32_t)(ubytes * 8);
            s.img = i; s.first_mcu = (long long)k * R; s.n_mcu = (int)std::min<long long>(R, d.nmcu - s.first_mcu);
            s.nsub = std::max<int>(1, (int)((s.b1 - s.b0 + JD_SUB - 1) / JD_SUB)); s.first_sub = 0;
            segs.push_back(s);
        }
        if (ubytes != u) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: inconsistent scan walk", i);
        if (in_bytes >= (1ull << 29)) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "decode_jpeg_batch: more than 512 MB of entropy-coded data in one call");
    }
    int nsub = 0;
    for (auto& s : segs) { s.first_sub = nsub; nsub += s.nsub; }
    std::vector<int> sub_seg(nsub);
    for (size_t k = 0; k < segs.size(); ++k)
        for (int j = 0; j < segs[k].nsub; ++j) sub_seg[segs[k].first_sub + j] = (int)k;
    const int nseg = (int)segs.size(), nchunk = (int)chunks.size();

    // ---- the upload: tables and layout, then the entropy-coded bytes
    const size_t o_tabs = 0, o_qt = o_tabs + al256(sizeof(JmHuff) * 8 * n), o_img = o_qt + al256(sizeof(int16_t) * 192 * n);
    const size_t o_seg = o_img + al256(sizeof(JdImg) * n), o_sub = o_seg + al256(sizeof(JdSeg) * nseg);
    const size_t o_chunk = o_sub + al256(sizeof(int) * nsub), o_in = o_chunk + al256(sizeof(JdChunk) * nchunk);
    const size_t o_rzimg = o_in + al256(in_bytes + 8), o_rztap = o_rzimg + al256(sizeof(RzImg) * rz.size());
    const size_t up_bytes = o_rztap + al256(sizeof(RzTap) * taps.size());
    SFM_CUDA(ctx, ctx->jpeg_pin_up.reserve(up_bytes));
    char* up = (char*)ctx->jpeg_pin_up.p;
    pool.parallel_for(n, [&](int i) {
        memcpy(up + o_tabs + sizeof(JmHuff) * 8 * i, ims[i].tabs, sizeof(JmHuff) * 8);
        memcpy(up + o_qt + sizeof(int16_t) * 192 * i, ims[i].qt, sizeof(int16_t) * 192);
        memcpy(up + o_in + in0[i], data[i] + ims[i].scan_off, ims[i].scan_len);
    });
    memcpy(up + o_img, img.data(), sizeof(JdImg) * n);
    memcpy(up + o_seg, segs.data(), sizeof(JdSeg) * nseg);
    memcpy(up + o_sub, sub_seg.data(), sizeof(int) * nsub);
    memcpy(up + o_chunk, chunks.data(), sizeof(JdChunk) * nchunk);
    memset(up + o_in + in_bytes, 0, 8);
    if (scaled) {
        memcpy(up + o_rzimg, rz.data(), sizeof(RzImg) * n);
        memcpy(up + o_rztap, taps.data(), sizeof(RzTap) * taps.size());
    }

    // ---- device memory
    const size_t o_down = al256(up_bytes);
    const size_t o_err = 0, o_stats = al256(sizeof(int) * n), o_out = o_stats + al256(sizeof(JdStats));
    const size_t down_bytes = o_out + (size_t)(scaled ? rzb : outb);
    const size_t o_u = o_down + al256(down_bytes), o_exit = o_u + al256(ubytes + 16);
    const size_t o_comp = o_exit + al256(8ull * nsub), o_chg = o_comp + al256(4ull * nsub), o_nblk = o_chg + al256(4ull * nsub);
    const size_t o_pre = o_nblk + al256(4ull * nsub), o_part = o_pre + al256(4ull * nsub);
    const size_t o_rc = o_part + al256(8ull * (ceil_div64(std::max<long long>(nsub, mcus), SCAN_TILE) + 1));
    const size_t o_msum = o_rc + 256, o_mpre = o_msum + al256(8ull * mcus);
    const size_t o_coef = o_mpre + al256(8ull * mcus), o_planes = o_coef + al256(128ull * blocks);
    const size_t o_full = o_planes + al256((size_t)planes);          // the decoded images of a scaled call (not downloaded)
    const size_t total = o_full + (scaled ? (size_t)outb : 0);
    SFM_CUDA(ctx, ctx->jpeg_dev.reserve(total));
    char* dv = (char*)ctx->jpeg_dev.p;
    const JmHuff* d_tabs = (const JmHuff*)(dv + o_tabs);
    const int16_t* d_qt = (const int16_t*)(dv + o_qt);
    const JdImg* d_img = (const JdImg*)(dv + o_img);
    const JdSeg* d_seg = (const JdSeg*)(dv + o_seg);
    const int* d_sub = (const int*)(dv + o_sub);
    const JdChunk* d_chunk = (const JdChunk*)(dv + o_chunk);
    const uint8_t* d_in = (const uint8_t*)(dv + o_in);
    char* down = dv + o_down;
    int* d_err = (int*)(down + o_err);
    JdStats* d_stats = (JdStats*)(down + o_stats);
    uint8_t* d_out = (uint8_t*)(down + o_out);
    uint8_t* d_u = (uint8_t*)(dv + o_u);
    uint64_t* d_exit = (uint64_t*)(dv + o_exit);
    int* d_comp = (int*)(dv + o_comp); int* d_chg = (int*)(dv + o_chg);
    uint32_t* d_nblk = (uint32_t*)(dv + o_nblk); uint32_t* d_pre = (uint32_t*)(dv + o_pre);
    void* d_part = dv + o_part;
    int* d_rc = (int*)(dv + o_rc);
    unsigned long long* d_msum = (unsigned long long*)(dv + o_msum); unsigned long long* d_mpre = (unsigned long long*)(dv + o_mpre);
    int16_t* d_coef = (int16_t*)(dv + o_coef);
    uint8_t* d_planes = (uint8_t*)(dv + o_planes);
    uint8_t* d_full = scaled ? (uint8_t*)(dv + o_full) : d_out;
    cudaStream_t st = ctx->stream;

    SFM_CUDA(ctx, cudaMemcpyAsync(dv, up, up_bytes, cudaMemcpyHostToDevice, st));
    SFM_CUDA(ctx, cudaMemsetAsync(down, 0, o_out, st));
    SFM_CUDA(ctx, cudaMemsetAsync(d_u + ubytes, 0, 16, st));
    SFM_CUDA(ctx, cudaMemsetAsync(d_rc, 0, 256, st));
    SFM_CUDA(ctx, cudaMemsetAsync(d_coef, 0, 128ull * blocks, st));
    jd_unstuff<<<nchunk, 256, 0, st>>>(d_in, d_chunk, d_u);
    SFM_LAUNCH_CHECK(ctx);
    const int sb = ceil_div(nsub, 128);
    jd_sync0<<<sb, 128, 0, st>>>(d_u, d_seg, d_sub, d_img, d_tabs, nsub, d_exit, d_comp, d_chg, d_stats);
    SFM_LAUNCH_CHECK(ctx);
    for (int r = 1; r <= JD_ROUNDS; ++r) {
        jd_sync_round<<<sb, 128, 0, st>>>(d_u, d_seg, d_sub, d_img, d_tabs, nsub, d_exit, d_comp, d_chg, d_rc, r, d_stats);
        SFM_LAUNCH_CHECK(ctx);
    }
    jd_sync_sweep<<<ceil_div(nseg, 4), 128, 0, st>>>(d_u, d_seg, nseg, d_img, d_tabs, d_exit, d_comp, d_chg, d_rc, d_stats);
    SFM_LAUNCH_CHECK(ctx);
    jd_nblk<<<sb, 128, 0, st>>>(d_exit, nsub, d_nblk);
    SFM_LAUNCH_CHECK(ctx);
    if (int rc = excl_scan<AddU32>(ctx, d_nblk, nsub, (uint32_t*)d_part, d_pre)) return rc;
    jd_write<<<sb, 128, 0, st>>>(d_u, d_seg, d_sub, d_img, d_tabs, nsub, d_exit, d_pre, d_coef, d_err);
    SFM_LAUNCH_CHECK(ctx);
    long long max_mcu = 0, max_blk = 0, max_pix = 0;
    for (auto& d : img) { max_mcu = std::max(max_mcu, d.nmcu); max_blk = std::max(max_blk, d.nblocks); max_pix = std::max(max_pix, (long long)d.OW * d.OH); }
    const dim3 gm((unsigned)ceil_div64(max_mcu, 128), (unsigned)n);
    jd_dc_sum<<<gm, 128, 0, st>>>(d_img, d_coef, d_msum);
    SFM_LAUNCH_CHECK(ctx);
    if (int rc = excl_scan<Add3x16>(ctx, d_msum, mcus, (unsigned long long*)d_part, d_mpre)) return rc;
    jd_dc_apply<<<gm, 128, 0, st>>>(d_img, d_coef, d_mpre);
    SFM_LAUNCH_CHECK(ctx);
    jd_idct<<<dim3((unsigned)ceil_div64(max_blk, 32), (unsigned)n), 256, 0, st>>>(d_img, d_coef, d_qt, d_planes);
    SFM_LAUNCH_CHECK(ctx);
    jd_color<<<dim3((unsigned)ceil_div64(max_pix, 256), (unsigned)n), 256, 0, st>>>(d_img, d_planes, d_full);
    SFM_LAUNCH_CHECK(ctx);
    if (scaled)
        if (int rc = rz_enqueue(ctx, scale, rz.data(), n, (const RzImg*)(dv + o_rzimg), (const RzTap*)(dv + o_rztap), d_full, d_out)) return rc;
    SFM_CUDA(ctx, ctx->jpeg_pin_down.reserve(down_bytes));
    char* hd = (char*)ctx->jpeg_pin_down.p;
    SFM_CUDA(ctx, cudaMemcpyAsync(hd, down, down_bytes, cudaMemcpyDeviceToHost, st));
    SFM_CUDA(ctx, cudaStreamSynchronize(st));

    const JdStats* hs = (const JdStats*)(hd + o_stats);
    ctx->jpeg_stats[0] = nsub; ctx->jpeg_stats[1] = hs->cw_first; ctx->jpeg_stats[2] = hs->cw_extra;
    ctx->jpeg_stats[3] = hs->rounds; ctx->jpeg_stats[4] = hs->swept;
    ctx->jpeg_stats[5] = (int64_t)up_bytes; ctx->jpeg_stats[6] = (int64_t)down_bytes;
    const int* herr = (const int*)(hd + o_err);
    for (int i = 0; i < n; ++i)
        if (herr[i])
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "image %d: %s", i,
                                herr[i] & JD_ERR_DATA ? "corrupt entropy-coded data (no Huffman code, overrun or a run past coefficient 63)"
                                                      : "entropy-coded data ends before the last block");
    pool.parallel_for(n, [&](int i) {
        const int ow = scaled ? rz[i].dw : img[i].OW, oh = scaled ? rz[i].dh : img[i].OH;
        const size_t row = (size_t)ow * 3, stride = out_stride && out_stride[i] ? out_stride[i] : row;
        const uint8_t* src = (const uint8_t*)(hd + o_out + (scaled ? rz[i].dst0 : img[i].out0));
        if (stride == row) memcpy(out_bgr[i], src, row * oh);
        else for (int y = 0; y < oh; ++y) memcpy(out_bgr[i] + y * stride, src + y * row, row);
    });
    return SFMB200_OK;
}

extern "C" {

int sfmb200_jpeg_info(const uint8_t* data, size_t size, int* width, int* height, int* components) {
    JpImage im; std::string why;
    const int rc = jp_parse(data, size, JD_CHUNK, im, why);
    if (rc) return rc;
    if (width) *width = im.OW;
    if (height) *height = im.OH;
    if (components) *components = im.ncomp;
    return SFMB200_OK;
}

int sfmb200_jpeg_last_stats(const sfmb200_ctx* ctx, int64_t* stats7) {
    if (!ctx || !stats7) return SFMB200_ERR_INVALID;
    for (int i = 0; i < 7; ++i) stats7[i] = ctx->jpeg_stats[i];
    return SFMB200_OK;
}

int sfmb200_decode_jpeg_batch(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, uint8_t* const* out_bgr,
                              const size_t* out_stride) {
    return jd_decode(ctx, data, size, n, 1.0, out_bgr, out_stride);
}

int sfmb200_decode_jpeg_batch_scaled(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale,
                                     uint8_t* const* out_bgr, const size_t* out_stride) {
    return jd_decode(ctx, data, size, n, scale, out_bgr, out_stride);
}

}  // extern "C"
