// match_tc.cu -- K1 on the Hopper tensor cores: knn2 as an exact integer GEMM (wgmma, s32 accumulators in registers), two
// instantiations.
//
// HAMMING (the reference's ORB case, SfM2DFeatureUtilities.cpp:39-40, 59-60).  For 256-bit descriptors
//   ham(q,t) = popc(q) + popc(t) - 2 <q,t>  with q,t in {0,1}^256 (SURVEY.md 8a-1); bits are mapped to SIGNED bytes +1/-1 so that
//   <a,b> = 256 - 2*hamming: wgmma.mma_async.m64n128k32.s32.s8.s8 (exact), 8 instructions per 64 x 128 accumulator.
// L2 (BASELINE.json configs[3] wording: SIFT-128; cv::BFMatcher(NORM_L2)).  SIFT descriptors are integer-valued 0..255, so
//   |a-b|^2 = |a|^2 + |b|^2 - 2 <a,b>  with <a,b> <= 128*255^2 < 2^31 is EXACT in u8 x u8 -> s32: 4 instructions per accumulator;
//   the train norms ride along in shared memory, the epilogue ranks  e = |b|^2 - 2<a,b>  (as packed keys e * 128 + column, one
//   multiply-add per element, see l2_group) and adds |a|^2 at the end.
//
//   * operands: expanded ONCE per descriptor set (expand kernels) into blocks of 256 rows in the GMMA K-major, no-swizzle
//     ("interleave") canonical form: core matrix = 8 rows x 16 bytes, LBO = distance between the 16-byte K chunks, SBO =
//     distance between 8-row groups (cute/arch/mma_sm90_desc.hpp, make_gmma_desc<Major::K>).  A tile travels HBM -> shared
//     memory as plain cp.async.bulk copies completing on an mbarrier (no tensor map needed: a block is contiguous).
//   * CTA = 128 query rows x one 256-row train tile per step: a loader warp and four consumer warpgroups, one per (64-row half,
//     128-column half) of the tile.  A warpgroup issues its wgmmas straight from shared memory, waits for them, releases the
//     B stage and ranks its 64 accumulators per thread while the other warpgroups' wgmmas run.
//   * accumulator fragment of m64nNk32 (PTX ISA, "wgmma register fragment D"): thread l of warp w of the warpgroup holds rows
//     16w + l/4 + {0, 8} and per row the columns 8j + 2(l%4) + {0, 1}, j < 16.  Every thread keeps a running top-2 per row; the
//     four threads of a row and the two column halves are merged at the end.
//   * Hamming keeps the running top-2 as two PACKED KEYS  key = (256 - 2 ham) << 16 | (0xFFFF - index)  -- larger is better, ties
//     go to the lower index exactly like cv::batchDistance -- so an insert is a 3-instruction max/min network (no compare/select
//     chains, no separate index registers), groups of 8 columns are skipped when no lane's group maximum (3-input max, DPX) beats
//     its second best.
// Bit-exact against the XOR/POPC kernel, the oracle and cv2 (tests/test_gpu_match.py); same merge / ratio / compaction epilogue.
#include "common.cuh"
#include "match_common.cuh"

namespace {

constexpr int TC_M = 128;            // query rows per CTA (two warpgroups of wgmma M = 64)
constexpr int TC_N = 256;            // train rows per tile = rows per expanded block
constexpr int TC_WN = 128;           // columns of the tile per consumer warpgroup (wgmma N)
constexpr int TC_CONSUMER_WARPS = 16;                    // 4 warpgroups: (row half, column half) of the 128 x 256 tile
constexpr int TC_THREADS = (TC_CONSUMER_WARPS + 1) * 32; // + warp 16: loader
constexpr int TC_NORM_SLOTS = 6;     // L2: ring of train-norm tiles (1 KB each); a slot is reused 6 tiles later, when its epilogue is long done

template <bool L2> struct TcCfg {
    static constexpr int KB = L2 ? 128 : 256;                  // operand bytes per row = K elements
    static constexpr int BLOCK_BYTES = TC_N * KB;              // one 256-row block of expanded operands
    static constexpr int A_BYTES = TC_M * KB;
    static constexpr int BSTAGES = L2 ? 4 : 3;                 // shared-memory stages of the train operand
    static constexpr int NORM_BYTES = L2 ? TC_NORM_SLOTS * TC_N * 4 : 0;
    static constexpr int HALF_BYTES = TC_M * 16;               // top-2 of the upper column half, one int4 per query row
    static constexpr int SMEM = A_BYTES + BSTAGES * BLOCK_BYTES + NORM_BYTES + HALF_BYTES + 256;
};
static_assert(TcCfg<false>::SMEM <= 227 * 1024, "Hamming pipeline exceeds the 227 KB of shared memory a block may use");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma shared-memory matrix descriptor, K-major, no swizzle (layout type 0, base offset 0):
// start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}

// 16 descriptor bits -> 16 signed bytes: bit 1 -> +1, bit 0 -> -1   (sum over k of a_k b_k = 256 - 2 * hamming)
__device__ __forceinline__ uint32_t pm1(uint32_t nib) {
    const uint32_t x = (nib * 0x00204081u) & 0x01010101u;
    return x | ((x ^ 0x01010101u) * 0xFFu);
}
__device__ __forceinline__ uint4 expand16(uint32_t bits16) {
    return make_uint4(pm1(bits16 & 0xF), pm1((bits16 >> 4) & 0xF), pm1((bits16 >> 8) & 0xF), pm1((bits16 >> 12) & 0xF));
}

// Expanded operand store (built once per descriptor set): per 256-row block the GMMA K-major no-swizzle canonical layout
//   [16-byte K chunk kc][row group r/8][r%8][16 B]   ->  LBO = 4096 B between K chunks, SBO = 128 B between 8-row groups.
// A 128-row half of a block is the same layout at start offset +2048 B per chunk, so one store serves both the query (M=128)
// and the train (N=256) operand.  Rows beyond the image are zero (contribute nothing).
__global__ void __launch_bounds__(256) expand_blocks_kernel(const uint32_t* __restrict__ desc, const int2* __restrict__ blocks /* (first row, valid rows) */,
                                                            uint8_t* __restrict__ E) {
    const int2 b = blocks[blockIdx.x];
    uint8_t* out = E + (size_t)blockIdx.x * TcCfg<false>::BLOCK_BYTES;
    for (int it = threadIdx.x; it < TC_N * 8; it += 256) {
        const int w = it / TC_N, r = it - w * TC_N;
        const bool valid = r < b.y;
        const uint32_t v = valid ? __ldg(desc + (size_t)(b.x + r) * 8 + w) : 0u;
        const uint4 lo = valid ? expand16(v & 0xFFFFu) : make_uint4(0, 0, 0, 0), hi = valid ? expand16(v >> 16) : make_uint4(0, 0, 0, 0);
        const uint32_t off = (uint32_t)(r >> 3) * 128 + (uint32_t)(r & 7) * 16;
        *reinterpret_cast<uint4*>(out + (size_t)(2 * w) * (TC_N * 16) + off) = lo;
        *reinterpret_cast<uint4*>(out + (size_t)(2 * w + 1) * (TC_N * 16) + off) = hi;
    }
}
// L2: float descriptors [rows][dim] (dim <= 128, zero-padded to 128) -> u8 operand blocks + squared norms.  *bad is raised when
// a value is not an integer in [0, 255] (then the exact-GEMM formulation does not apply and the caller falls back to fp32).
__global__ void __launch_bounds__(256) expand_l2_blocks_kernel(const float* __restrict__ desc, int dim, const int2* __restrict__ blocks,
                                                               uint8_t* __restrict__ E, int32_t* __restrict__ norms, int* __restrict__ bad) {
    const int2 b = blocks[blockIdx.x];
    uint8_t* out = E + (size_t)blockIdx.x * TcCfg<true>::BLOCK_BYTES;
    const int r = threadIdx.x;                                              // one row per thread
    const bool valid = r < b.y;
    const float* src = desc + (size_t)(b.x + (valid ? r : 0)) * dim;
    int nrm = 0; bool ok = true;
    const uint32_t off = (uint32_t)(r >> 3) * 128 + (uint32_t)(r & 7) * 16;
    for (int kc = 0; kc < 8; ++kc) {
        uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int k = kc * 16 + j;
            float f = (valid && k < dim) ? __ldg(src + k) : 0.f;
            const int iv = (int)f;
            ok = ok && (f == (float)iv) && iv >= 0 && iv <= 255;
            const int c = min(max(iv, 0), 255);
            nrm += c * c;
            w[j >> 2] |= (uint32_t)c << (8 * (j & 3));
        }
        *reinterpret_cast<uint4*>(out + (size_t)kc * (TC_N * 16) + off) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    // packed for the epilogue's key arithmetic: |b|^2 * 128 + (row & 127: the column inside its 128-column half of the tile); |b|^2 <= 128 * 255^2 < 2^23
    norms[(size_t)blockIdx.x * TC_N + r] = ((valid ? nrm : 0) << 7) | (r & 127);
    if (!ok) atomicExch(bad, 1);
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %0;" ::"r"(bytes), "r"(smem_u32(bar)) : "memory"); }
// bounded wait: returns false if the barrier never flips (a descriptor mistake must not hang the GPU)
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    for (int spin = 0; spin < (1 << 22); ++spin) {
        uint32_t done;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return true;
    }
    return false;
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes),
                 "r"(smem_u32(bar)) : "memory");
}
// AND of p over the 128 threads of a warpgroup (named barrier `id`): keeps the early exit of a timed-out wait warpgroup-uniform,
// which the .sync.aligned wgmma instructions require
__device__ __forceinline__ bool wg_all(bool p, int id) {
    uint32_t r;
    asm volatile("{ .reg .pred a, b; setp.ne.u32 a, %1, 0; bar.red.and.pred b, %2, 128, a; selp.u32 %0, 1, 0, b; }" : "=r"(r) : "r"((uint32_t)p), "r"(id) : "memory");
    return r != 0;
}

#define TC_ACC_REGS "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
                    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
                    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define TC_ACC8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
#define TC_ACC_OPS TC_ACC8(0), TC_ACC8(8), TC_ACC8(16), TC_ACC8(24), TC_ACC8(32), TC_ACC8(40), TC_ACC8(48), TC_ACC8(56)

// one m64n128k32 integer wgmma: d (+)= A[64 x 32] * B[128 x 32]^T, s8 x s8 (Hamming) or u8 x u8 (L2) -> s32
template <bool L2> __device__ __forceinline__ void wgmma_i8(uint32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if (L2)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 " TC_ACC_REGS ", %64, %65, p;\n\t}\n"
                     : TC_ACC_OPS : "l"(adesc), "l"(bdesc), "r"(accumulate) : "memory");
    else
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " TC_ACC_REGS ", %64, %65, p;\n\t}\n"
                     : TC_ACC_OPS : "l"(adesc), "l"(bdesc), "r"(accumulate) : "memory");
}
// the accumulators are written asynchronously until wgmma.wait_group: the empty asm pins every read of them after the wait
__device__ __forceinline__ void acc_fence(uint32_t (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// Hamming key: (256 - 2 ham) in the high half, 0xFFFF - (train index inside this CTA's split) in the low half.  The split of a
// CTA covers at most 256 tiles = 65536 rows (match_tc_splits), so the index fits.  EMPTY = INT_MIN sorts below every key.
constexpr int KEY_EMPTY = INT_MIN;

// acc register of (row r of the thread's two, column pair j, element e of the pair)
__device__ __forceinline__ int acc_at(const uint32_t (&d)[64], int r, int j, int e) { return (int)d[4 * j + 2 * r + e]; }

// One group of 8 columns (pairs j = 4g..4g+3) of row r of the Hamming epilogue.  v = 256 - 2 ham.  A 3-input-max tree, one vote,
// and -- only when SOME lane of the warp has a candidate above its second best -- the insert network on packed keys:
// {k0, k1, key} -> the two largest.  cb = low key half of this thread's column 0; column of (j, e) = 8j + e past it.
// PART: columns >= ncols (counted from this thread's column 0) are zero padding of the image's last tile.
template <bool PART>
__device__ __forceinline__ void hamming_group(const uint32_t (&d)[64], int r, int g, int cb, int ncols, int& k0, int& k1, int& thr) {
    int m = __vimax3_s32(acc_at(d, r, 4 * g, 0), acc_at(d, r, 4 * g, 1), acc_at(d, r, 4 * g + 1, 0));
    m = __vimax3_s32(m, acc_at(d, r, 4 * g + 1, 1), acc_at(d, r, 4 * g + 2, 0));
    m = __vimax3_s32(m, acc_at(d, r, 4 * g + 2, 1), acc_at(d, r, 4 * g + 3, 0));
    m = max(m, acc_at(d, r, 4 * g + 3, 1));
    if (PART || __any_sync(0xffffffffu, m > thr)) {
#pragma unroll
        for (int j = 4 * g; j < 4 * g + 4; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                int key = acc_at(d, r, j, e) * 65536 + (cb - 8 * j - e);
                if (PART && 8 * j + e >= ncols) key = KEY_EMPTY;
                const int hi = max(k0, key), lo = min(k0, key);
                k1 = max(k1, lo); k0 = hi;
            }
        thr = k1 >> 16;                 // a later candidate needs a strictly larger v: with equal v its index loses
    }
}

// L2 key: e * 128 + (column inside the 128-column half of the tile), e = |b|^2 - 2<a,b> in [-2 * 128 * 255^2, 128 * 255^2] -- 25 bits, so the key
// fits a signed 32-bit word exactly and ONE multiply-add makes it from the accumulator: key = nk - (acc << 8) with the packed norm
// nk = |b|^2 * 128 + column that rides along in shared memory.  Smaller key = smaller distance, ties to the smaller column: the order
// of cv::batchDistance inside a tile.  The keys only live for one tile (7 index bits): per 8-column group a 3-input-min tree and a
// vote against thrk (the running second best of the row as a key bound, tightened by the tile's own second best), then the
// {k0, k1, key} -> two smallest network; after the tile the two survivors are unpacked and merged into the (distance, index) pairs.
// nk points at the packed norm of this thread's column 0.
constexpr int L2KEY_EMPTY = INT_MAX;
template <bool PART>
__device__ __forceinline__ void l2_group(const uint32_t (&d)[64], int r, int g, const int32_t* __restrict__ nk, int ncols, int& k0, int& k1, int& thrk) {
    int key[8];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * g + jj;
        const int2 n = *reinterpret_cast<const int2*>(nk + 8 * j);
        key[2 * jj] = n.x - (acc_at(d, r, j, 0) << 8);
        key[2 * jj + 1] = n.y - (acc_at(d, r, j, 1) << 8);
        if (PART && 8 * j >= ncols) key[2 * jj] = L2KEY_EMPTY;
        if (PART && 8 * j + 1 >= ncols) key[2 * jj + 1] = L2KEY_EMPTY;
    }
    int m = __vimin3_s32(key[0], key[1], key[2]);
    m = __vimin3_s32(m, key[3], key[4]); m = __vimin3_s32(m, key[5], key[6]); m = min(m, key[7]);
    if (PART || __any_sync(0xffffffffu, m < thrk)) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int lo = min(k0, key[j]), hi = max(k0, key[j]);
            k1 = min(k1, hi); k0 = lo;
        }
        thrk = min(thrk, k1);
    }
}

// lexicographic (distance, index) top-2 insert; index < 0 = empty
__device__ __forceinline__ void lex_insert(Top2& b, int d, int i) {
    auto lt = [](int d1, int i1, int d2, int i2) { return d1 < d2 || (d1 == d2 && i1 < i2); };
    if (i < 0) return;
    if (b.i0 < 0 || lt(d, i, b.d0, b.i0)) { b.d1 = b.d0; b.i1 = b.i0; b.d0 = d; b.i0 = i; }
    else if (b.i1 < 0 || lt(d, i, b.d1, b.i1)) { b.d1 = d; b.i1 = i; }
}

// Warp-specialised: loader thread (cp.async.bulk of pre-expanded blocks) -> four consumer warpgroups (wgmma from shared memory
// into 64 registers per thread, then the running top-2 per query row in registers).
template <bool L2>
__global__ void __launch_bounds__(TC_THREADS, 1) knn2_tc_kernel(const uint8_t* __restrict__ E, const int32_t* __restrict__ norms, const PairDesc* __restrict__ pairs,
                                                                int qblocks, int splits, int4* __restrict__ partial, int* __restrict__ error_flag) {
    using C = TcCfg<L2>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sA = smem;
    uint8_t* sB = smem + C::A_BYTES;
    int32_t* sNorm = reinterpret_cast<int32_t*>(smem + C::A_BYTES + C::BSTAGES * C::BLOCK_BYTES);      // [TC_NORM_SLOTS][TC_N]   (L2)
    int4* half_best = reinterpret_cast<int4*>(smem + C::A_BYTES + C::BSTAGES * C::BLOCK_BYTES + C::NORM_BYTES);   // [TC_M]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::A_BYTES + C::BSTAGES * C::BLOCK_BYTES + C::NORM_BYTES + C::HALF_BYTES);
    uint64_t* a_full = bars;                 // [1]
    uint64_t* full = bars + 1;               // [BSTAGES] bytes of a B stage have landed
    uint64_t* smem_free = full + C::BSTAGES; // [BSTAGES] the wgmmas of every consumer warp that read the stage have completed

    const PairDesc pd = pairs[blockIdx.y];
    const int qb = blockIdx.x / splits, sp = blockIdx.x % splits;
    if (qb * TC_M >= pd.nq) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_total = (pd.nt + TC_N - 1) / TC_N;
    const int tiles_per_split = (tiles_total + splits - 1) / splits;
    const int tile0 = sp * tiles_per_split, ntiles = max(0, min(tiles_total, tile0 + tiles_per_split) - tile0);
    const int q_row0 = qb * TC_M;

    if (threadIdx.x == 0) {
        mbar_init(a_full, 1);
        for (int i = 0; i < C::BSTAGES; ++i) { mbar_init(full + i, 1); mbar_init(smem_free + i, TC_CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    bool ok = true;

    // consumer geometry: warpgroup wg = (row half rh, column half ch); this thread's rows (of the CTA's 128) and column 0 (of the
    // warpgroup's 128) in the accumulator fragment
    const int wg = warp >> 2, rh = wg & 1, ch = wg >> 1;
    const int row_a = rh * 64 + (warp & 3) * 16 + (lane >> 2), col0 = 2 * (lane & 3);
    // Hamming: packed keys per row; L2: (e = |b|^2 - 2<a,b>, global index) pairs per row
    int k0[2] = {KEY_EMPTY, KEY_EMPTY}, k1[2] = {KEY_EMPTY, KEY_EMPTY};
    Top2 best[2] = {{INT_MAX, -1, INT_MAX, -1}, {INT_MAX, -1, INT_MAX, -1}};
    if (warp == TC_CONSUMER_WARPS) {
        if (lane == 0) {
            // ---- loader: query tile (a 128-row half of a block: KB/16 chunks of 2 KB), then the train blocks (+ their norms)
            const uint8_t* qsrc = E + (size_t)(pd.q_blk + q_row0 / TC_N) * C::BLOCK_BYTES + (size_t)((q_row0 / TC_M) & 1) * (TC_M * 16);
            mbar_expect_tx(a_full, C::A_BYTES);
            for (int kc = 0; kc < C::KB / 16; ++kc) bulk_g2s(sA + kc * (TC_M * 16), qsrc + (size_t)kc * (TC_N * 16), TC_M * 16, a_full);
            for (int t = 0; t < ntiles && ok; ++t) {
                const int s = t % C::BSTAGES, u = t / C::BSTAGES;
                if (u > 0 && !mbar_wait(smem_free + s, (u - 1) & 1)) { ok = false; break; }
                const uint8_t* src = E + (size_t)(pd.t_blk + tile0 + t) * C::BLOCK_BYTES;
                mbar_expect_tx(full + s, C::BLOCK_BYTES + (L2 ? TC_N * 4 : 0));
                for (int c = 0; c < 4; ++c) bulk_g2s(sB + s * C::BLOCK_BYTES + c * (C::BLOCK_BYTES / 4), src + c * (C::BLOCK_BYTES / 4), C::BLOCK_BYTES / 4, full + s);
                if (L2) bulk_g2s(sNorm + (t % TC_NORM_SLOTS) * TC_N, norms + (size_t)(pd.t_blk + tile0 + t) * TC_N, TC_N * 4, full + s);
            }
        }
    } else {
        // ---- consumer warpgroups.  The query tile always lands before the CTA exits (also when the split owns no train tile).
        ok = wg_all(mbar_wait(a_full, 0), 1 + wg);
        // A: rows 64*rh.. of the query tile (8 row groups of 128 B past the tile start); B: columns 128*ch.. of the stage
        const uint32_t a0 = smem_u32(sA) + (uint32_t)rh * 8 * 128;
        int thr[2] = {L2 ? INT_MAX : INT_MIN, L2 ? INT_MAX : INT_MIN};    // Hamming: v must exceed it; L2: the key must be below it
        uint32_t d[64] = {};
        for (int t = 0; t < ntiles && ok; ++t) {
            const int s = t % C::BSTAGES, u = t / C::BSTAGES;
            if (!(ok = wg_all(mbar_wait(full + s, u & 1), 1 + wg))) break;
            const uint32_t b0 = smem_u32(sB + s * C::BLOCK_BYTES) + (uint32_t)ch * 16 * 128;
            acc_fence(d);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int kk = 0; kk < C::KB / 32; ++kk) {                // K = 32 bytes per instruction = two 16-byte chunks
                const uint64_t ad = make_smem_desc(a0 + 2 * kk * (TC_M * 16), TC_M * 16, 128);
                const uint64_t bd = make_smem_desc(b0 + 2 * kk * (TC_N * 16), TC_N * 16, 128);
                wgmma_i8<L2>(d, ad, bd, kk > 0 ? 1u : 0u);
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            acc_fence(d);
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_free + s);             // this warp's reads of the B stage are complete

            const int t_row0 = (tile0 + t) * TC_N, ncols = min(TC_N, pd.nt - t_row0) - ch * TC_WN - col0;   // real columns past this thread's column 0
            if (min(TC_N, pd.nt - t_row0) <= ch * TC_WN) continue;            // this column half is all padding (warpgroup-uniform)
            const bool part = min(TC_N, pd.nt - t_row0) < (ch + 1) * TC_WN;  // last tile of the image only
            if (!L2) {
                const int cb = 0xFFFF - (t * TC_N + ch * TC_WN + col0);       // low key half of this thread's column 0
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        if (!part) hamming_group<false>(d, r, g, cb, ncols, k0[r], k1[r], thr[r]);
                        else hamming_group<true>(d, r, g, cb, ncols, k0[r], k1[r], thr[r]);
                    }
            } else {
                const int32_t* nk = sNorm + (t % TC_NORM_SLOTS) * TC_N + ch * TC_WN + col0;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    int kt0 = L2KEY_EMPTY, kt1 = L2KEY_EMPTY;                // the tile's two smallest keys of this row
                    thr[r] = best[r].i1 < 0 ? INT_MAX : (best[r].d1 << 7);  // a later row must be STRICTLY closer than the running second best
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        if (!part) l2_group<false>(d, r, g, nk, ncols, kt0, kt1, thr[r]);
                        else l2_group<true>(d, r, g, nk, ncols, kt0, kt1, thr[r]);
                    }
                    // the tile's survivors -> (e, global index), ascending key order; earlier tiles win ties
                    auto ins = [&](int key) {
                        if (key == L2KEY_EMPTY) return;
                        const int dd = key >> 7, idx = t_row0 + ch * TC_WN + (key & 127);
                        if (dd < best[r].d0) { best[r].d1 = best[r].d0; best[r].i1 = best[r].i0; best[r].d0 = dd; best[r].i0 = idx; }
                        else if (dd < best[r].d1) { best[r].d1 = dd; best[r].i1 = idx; }
                    };
                    ins(kt0); ins(kt1);
                }
            }
        }
        // merge the four threads of each row (lanes 4k..4k+3)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int off = 1; off < 4; off <<= 1) {
                if (!L2) {
                    const int o0 = __shfl_xor_sync(0xffffffffu, k0[r], off), o1 = __shfl_xor_sync(0xffffffffu, k1[r], off);
                    int hi = max(k0[r], o0), lo = min(k0[r], o0); k1[r] = max(k1[r], lo); k0[r] = hi;
                    hi = max(k0[r], o1); lo = min(k0[r], o1); k1[r] = max(k1[r], lo); k0[r] = hi;
                } else {
                    const int d0 = __shfl_xor_sync(0xffffffffu, best[r].d0, off), i0 = __shfl_xor_sync(0xffffffffu, best[r].i0, off);
                    const int d1 = __shfl_xor_sync(0xffffffffu, best[r].d1, off), i1 = __shfl_xor_sync(0xffffffffu, best[r].i1, off);
                    lex_insert(best[r], d0, i0); lex_insert(best[r], d1, i1);
                }
            }
        if (ch == 1 && (lane & 3) == 0)
            for (int r = 0; r < 2; ++r)
                half_best[row_a + 8 * r] = L2 ? make_int4(best[r].d0, best[r].i0, best[r].d1, best[r].i1) : make_int4(k0[r], k1[r], 0, 0);
    }
    if (!ok) atomicExch(error_flag, 1);
    __syncthreads();
    if (warp < TC_CONSUMER_WARPS && ch == 0 && (lane & 3) == 0) {
        for (int r = 0; r < 2; ++r) {
            const int rloc = row_a + 8 * r, row = q_row0 + rloc;
            const int4 o = half_best[rloc];
            if (!L2) {
                // merge the column halves with the same network, then unpack
                int hi = max(k0[r], o.x), lo = min(k0[r], o.x); k1[r] = max(k1[r], lo); k0[r] = hi;
                hi = max(k0[r], o.y); lo = min(k0[r], o.y); k1[r] = max(k1[r], lo); k0[r] = hi;
                auto unpack = [&](int key, int& dd, int& i) {
                    if (key == KEY_EMPTY) { dd = INT_MAX; i = -1; return; }
                    dd = (256 - (key >> 16)) >> 1; i = tile0 * TC_N + (0xFFFF - (key & 0xFFFF));
                };
                int d0, i0, d1, i1; unpack(k0[r], d0, i0); unpack(k1[r], d1, i1);
                if (row < pd.nq) partial[(size_t)(pd.out_row + row) * splits + sp] = make_int4(d0, i0, d1, i1);
            } else {
                // lexicographic (e, index) merge, then |a|^2 + e = squared distance (exact integer)
                lex_insert(best[r], o.x, o.y); lex_insert(best[r], o.z, o.w);
                if (row < pd.nq) {
                    const int na = norms[(size_t)(pd.q_blk + q_row0 / TC_N) * TC_N + (q_row0 % TC_N) + rloc] >> 7;      // packed: |a|^2 * 128 + column
                    partial[(size_t)(pd.out_row + row) * splits + sp] =
                        make_int4(best[r].i0 >= 0 ? na + best[r].d0 : INT_MAX, best[r].i0, best[r].i1 >= 0 ? na + best[r].d1 : INT_MAX, best[r].i1);
                }
            }
        }
    }
}

}  // namespace

int match_tc_splits(int sm_count, int n_pairs, int nq_max, int nt_max) {
    const int qblocks = ceil_div(nq_max, TC_M), tiles = ceil_div(nt_max, TC_N);
    int splits = 1;
    while ((int64_t)qblocks * n_pairs * splits < 2LL * sm_count && splits * 2 <= tiles && splits < 16) splits *= 2;
    while (ceil_div(tiles, splits) > 256) splits *= 2;       // the 16-bit index field of the Hamming key: <= 256 tiles per split
    return splits;
}

size_t match_tc_block_bytes(bool l2) { return l2 ? TcCfg<true>::BLOCK_BYTES : TcCfg<false>::BLOCK_BYTES; }
int match_tc_block_rows() { return TC_N; }

int match_tc_expand(sfmb200_ctx* ctx, const uint32_t* d_desc, const int2* d_blocks, int n_blocks, uint8_t* d_E) {
    if (n_blocks == 0) return SFMB200_OK;
    expand_blocks_kernel<<<n_blocks, 256, 0, ctx->stream>>>(d_desc, d_blocks, d_E);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}
int match_tc_expand_l2(sfmb200_ctx* ctx, const float* d_desc, int dim, const int2* d_blocks, int n_blocks, uint8_t* d_E, int32_t* d_norms, int* d_bad) {
    if (n_blocks == 0) return SFMB200_OK;
    expand_l2_blocks_kernel<<<n_blocks, 256, 0, ctx->stream>>>(d_desc, dim, d_blocks, d_E, d_norms, d_bad);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

int match_tc_launch(sfmb200_ctx* ctx, bool l2, const uint8_t* d_E, const int32_t* d_norms, const PairDesc* d_pairs, int n_pairs, int nq_max, int splits,
                    int4* d_partial, int* d_error_flag) {
    // the attribute is per device and the context is per device; ctx->mu is held by every caller
    if (!ctx->tc_attr_set) {
        SFM_CUDA(ctx, cudaFuncSetAttribute(knn2_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<false>::SMEM));
        SFM_CUDA(ctx, cudaFuncSetAttribute(knn2_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<true>::SMEM));
        ctx->tc_attr_set = true;
    }
    const int qblocks = ceil_div(nq_max, TC_M);
    dim3 grid(qblocks * splits, n_pairs);
    if (l2) knn2_tc_kernel<true><<<grid, TC_THREADS, TcCfg<true>::SMEM, ctx->stream>>>(d_E, d_norms, d_pairs, qblocks, splits, d_partial, d_error_flag);
    else knn2_tc_kernel<false><<<grid, TC_THREADS, TcCfg<false>::SMEM, ctx->stream>>>(d_E, d_norms, d_pairs, qblocks, splits, d_partial, d_error_flag);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}
