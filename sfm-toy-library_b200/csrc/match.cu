// match.cu -- K1: brute-force 2-nearest-neighbour descriptor matching with fused ratio test.
//
// Replaces SfM2DFeatureUtilities::matchFeatures (reference SfMToyLib/SfM2DFeatureUtilities.cpp:53-71):
//   cv::DescriptorMatcher("BruteForce-Hamming")->knnMatch(k=2)  (:59-60)  + ratio test d0 < (double)0.8f * d1 (:35, :65)
// and, batched over image pairs, the thread fan-out of SfM::createFeatureMatchMatrix (SfM.cpp:157-212).
//
// Integer path (bit-exact): XOR + POPC on 32-bit words, distance in int, ordering lexicographic on
// (distance, trainIdx) so that ties go to the lower train index like cv::batchDistance.
//
// Kernels
//   knn2_hamming_kernel<WORDS>  grid (qblocks*splits, pairs): each thread owns QPT query rows in registers; train rows are
//                               staged through shared memory in tiles (coalesced 16-byte loads, broadcast LDS.128 reads);
//                               top-2 per (query, train split) -> partial[].  The Nq x Nt distance matrix never exists.
//   merge_flag_scan_kernel      merges the splits in index order, applies the ratio test in double, block-scans the flags
//   scan_sums_kernel            exclusive scan of the per-block survivor counts (single CTA, chained)
//   scatter_kernel              order-preserving compaction into (queryIdx, trainIdx, distance) + per-pair counts
#include "common.cuh"
#include "match_common.cuh"
#include <cstdlib>

namespace {

constexpr int KNN_THREADS = 128;
constexpr int QPT = 2;                       // query rows per thread
constexpr int QBLOCK = KNN_THREADS * QPT;    // query rows per CTA
constexpr int TILE = 128;                    // train rows per shared-memory tile
constexpr int SCAN_THREADS = 1024;

template <int WORDS>
__global__ void __launch_bounds__(KNN_THREADS)
knn2_hamming_kernel(const uint32_t* __restrict__ desc, const PairDesc* __restrict__ pairs, int qblocks, int splits,
                    int4* __restrict__ partial) {
    __shared__ __align__(16) uint32_t tile[TILE * WORDS];
    const PairDesc pd = pairs[blockIdx.y];
    const int qb = blockIdx.x / splits, sp = blockIdx.x % splits;
    if (qb * QBLOCK >= pd.nq) return;
    // train rows of this split: [t_begin, t_end)
    const int chunk = (pd.nt + splits - 1) / splits;
    const int t_begin = sp * chunk, t_end = min(pd.nt, t_begin + chunk);

    uint32_t q[QPT][WORDS];
    Top2 best[QPT];
#pragma unroll
    for (int u = 0; u < QPT; ++u) {
        const int row = qb * QBLOCK + u * KNN_THREADS + threadIdx.x;
        best[u] = {INT_MAX, -1, INT_MAX, -1};
        const uint4* src = reinterpret_cast<const uint4*>(desc + (size_t)(pd.q_row + min(row, pd.nq - 1)) * WORDS);
#pragma unroll
        for (int w = 0; w < WORDS / 4; ++w) {
            const uint4 v = __ldg(src + w);
            q[u][4 * w] = v.x; q[u][4 * w + 1] = v.y; q[u][4 * w + 2] = v.z; q[u][4 * w + 3] = v.w;
        }
    }

    for (int t0 = t_begin; t0 < t_end; t0 += TILE) {
        const int rows = min(TILE, t_end - t0);
        __syncthreads();
        {   // stage `rows` train rows: rows*WORDS/4 uint4, coalesced
            const uint4* src = reinterpret_cast<const uint4*>(desc + (size_t)(pd.t_row + t0) * WORDS);
            uint4* dst = reinterpret_cast<uint4*>(tile);
            for (int i = threadIdx.x; i < rows * (WORDS / 4); i += KNN_THREADS) dst[i] = __ldg(src + i);
        }
        __syncthreads();
#pragma unroll 2
        for (int j = 0; j < rows; ++j) {
            const uint4* tr = reinterpret_cast<const uint4*>(tile + j * WORDS);
            int d[QPT];
#pragma unroll
            for (int u = 0; u < QPT; ++u) d[u] = 0;
#pragma unroll
            for (int w = 0; w < WORDS / 4; ++w) {
                const uint4 v = tr[w];                  // same address for the whole warp: one broadcast wavefront
#pragma unroll
                for (int u = 0; u < QPT; ++u)
                    d[u] += __popc(q[u][4 * w] ^ v.x) + __popc(q[u][4 * w + 1] ^ v.y) + __popc(q[u][4 * w + 2] ^ v.z) +
                            __popc(q[u][4 * w + 3] ^ v.w);
            }
#pragma unroll
            for (int u = 0; u < QPT; ++u) top2_insert(best[u], d[u], t0 + j);
        }
    }
#pragma unroll
    for (int u = 0; u < QPT; ++u) {
        const int row = qb * QBLOCK + u * KNN_THREADS + threadIdx.x;
        if (row < pd.nq) partial[(size_t)(pd.out_row + row) * splits + sp] = make_int4(best[u].d0, best[u].i0, best[u].d1, best[u].i1);
    }
}

// L2 (float) variant: one warp per query row, lanes split the dimension; squared distance accumulated in float32,
// sqrt in float (cv::BFMatcher(NORM_L2)).  Exact for integer-valued descriptors (sums < 2^24).
__global__ void __launch_bounds__(256)
knn2_l2_kernel(const float* __restrict__ q, int nq, const float* __restrict__ t, int nt, int dim, int splits, float4* __restrict__ partial) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int row = warp / splits, sp = warp % splits;
    if (row >= nq) return;
    const int chunk = (nt + splits - 1) / splits, t_begin = sp * chunk, t_end = min(nt, t_begin + chunk);
    float d0 = 3.4e38f, d1 = 3.4e38f; int i0 = -1, i1 = -1;
    for (int j = t_begin; j < t_end; ++j) {
        float s = 0.f;
        for (int k = lane; k < dim; k += 32) { const float e = q[(size_t)row * dim + k] - __ldg(t + (size_t)j * dim + k); s = fmaf(e, e, s); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (s < d0) { d1 = d0; i1 = i0; d0 = s; i0 = j; } else if (s < d1) { d1 = s; i1 = j; }
    }
    if (lane == 0) partial[(size_t)row * splits + sp] = make_float4(d0, __int_as_float(i0), d1, __int_as_float(i1));
}

// warp + block exclusive scan of one int per thread (SCAN_THREADS threads); returns exclusive prefix, total in *total
__device__ __forceinline__ int block_exclusive_scan(int v, int* total) {
    __shared__ int warp_sums[SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
    if (lane == 31) warp_sums[w] = inc;
    __syncthreads();
    if (w == 0) {
        int s = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += n; }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    const int base = w > 0 ? warp_sums[w - 1] : 0;
    *total = warp_sums[SCAN_THREADS / 32 - 1];
    return base + inc - v;
}

// rows = flattened query rows of all pairs.  is_l2: partials are float4 (squared distances)
__global__ void __launch_bounds__(SCAN_THREADS)
merge_flag_scan_kernel(const int4* __restrict__ partial, int splits, int64_t rows, double ratio, int is_l2,
                       int32_t* __restrict__ best_t, float* __restrict__ best_d, int32_t* __restrict__ rank,
                       uint8_t* __restrict__ flag, int32_t* __restrict__ block_sums) {
    const int64_t g = (int64_t)blockIdx.x * SCAN_THREADS + threadIdx.x;
    int keep = 0;
    if (g < rows) {
        float fd0, fd1; int i0 = -1, i1 = -1;
        if (is_l2 != 1) {
            Top2 b = {INT_MAX, -1, INT_MAX, -1};
            for (int s = 0; s < splits; ++s) {
                const int4 p = partial[(size_t)g * splits + s];
                if (p.y >= 0) top2_insert(b, p.x, p.y);
                if (p.w >= 0) top2_insert(b, p.z, p.w);
            }
            i0 = b.i0; i1 = b.i1; fd0 = (float)b.d0; fd1 = (float)b.d1;          // DMatch.distance is float
            // is_l2 == 2: exact integer SQUARED L2 distances (wgmma u8 GEMM); cv::batchDistance returns sqrt of the float sum
            if (is_l2 == 2) { fd0 = sqrtf(fd0); fd1 = sqrtf(fd1); }
        } else {
            float d0 = 3.4e38f, d1 = 3.4e38f;
            const float4* pf = reinterpret_cast<const float4*>(partial);
            for (int s = 0; s < splits; ++s) {
                const float4 p = pf[(size_t)g * splits + s];
                const int a = __float_as_int(p.y), c = __float_as_int(p.w);
                if (a >= 0) { if (p.x < d0) { d1 = d0; i1 = i0; d0 = p.x; i0 = a; } else if (p.x < d1) { d1 = p.x; i1 = a; } }
                if (c >= 0) { if (p.z < d0) { d1 = d0; i1 = i0; d0 = p.z; i0 = c; } else if (p.z < d1) { d1 = p.z; i1 = c; } }
            }
            fd0 = sqrtf(d0); fd1 = sqrtf(d1);
        }
        // reference: initialMatching[i][0].distance < NN_MATCH_RATIO * initialMatching[i][1].distance, in double (:65)
        keep = (i0 >= 0 && i1 >= 0) && ((double)fd0 < ratio * (double)fd1);
        best_t[g] = i0; best_d[g] = fd0; flag[g] = (uint8_t)keep;
    }
    int total;
    const int ex = block_exclusive_scan(keep, &total);
    if (g < rows) rank[g] = ex;
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// in-place exclusive scan of block_sums[n] (single CTA, chained over chunks); total -> *grand_total
__global__ void __launch_bounds__(SCAN_THREADS) scan_sums_kernel(int32_t* __restrict__ sums, int n, int64_t* __restrict__ grand_total,
                                                                 const int* __restrict__ error_flag /* may be null */) {
    __shared__ int carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n; base += SCAN_THREADS) {
        const int i = base + threadIdx.x;
        const int v = i < n ? sums[i] : 0;
        int total;
        const int ex = block_exclusive_scan(v, &total);
        const int carry = carry_s;
        if (i < n) sums[i] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + total;
        __syncthreads();
    }
    // a tensor-core pipeline error (bounded mbarrier wait expired) poisons the total: device-resident callers see -1
    if (threadIdx.x == 0) *grand_total = (error_flag && *error_flag) ? -1 : carry_s;
}

__global__ void __launch_bounds__(SCAN_THREADS)
scatter_kernel(const PairDesc* __restrict__ pairs, int n_pairs, int64_t rows, const int32_t* __restrict__ best_t,
               const float* __restrict__ best_d, const int32_t* __restrict__ rank, const uint8_t* __restrict__ flag,
               const int32_t* __restrict__ block_off, int32_t* __restrict__ out_q, int32_t* __restrict__ out_t,
               float* __restrict__ out_d, int32_t* __restrict__ pair_start /* [n_pairs+1] dense position of each pair's first survivor */) {
    const int64_t g = (int64_t)blockIdx.x * SCAN_THREADS + threadIdx.x;
    if (g >= rows) return;
    const int pos = block_off[blockIdx.x] + rank[g];
    // which pair does row g belong to?  binary search on out_row
    int lo = 0, hi = n_pairs - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (pairs[mid].out_row <= g) lo = mid; else hi = mid - 1; }
    const int local = (int)(g - pairs[lo].out_row);
    if (local == 0) pair_start[lo] = pos;
    if (flag[g]) { out_q[pos] = local; out_t[pos] = best_t[g]; out_d[pos] = best_d[g]; }
}

int choose_splits(int sm_count, int64_t ctas_without_split, int nt_max) {
    int s = 1;
    while (ctas_without_split * s < 4LL * sm_count && s < 32 && nt_max / (s * 2) >= TILE) s *= 2;
    return s;
}

}  // namespace

struct sfmb200_descset {
    sfmb200_ctx* ctx;
    uint32_t* d_desc = nullptr;
    std::vector<int32_t> img_off;
    int n_img = 0, words = 0, max_rows = 0;
    // tensor-core path (32-byte Hamming descriptors, u8-valued L2 descriptors): operands expanded once, blocks of 256 rows
    uint8_t* d_exp = nullptr;
    std::vector<int32_t> img_blk;      // first block of each image
    int kind = 0;                      // 0 = Hamming, 1 = L2 (exact u8 GEMM)
    int32_t* d_norms = nullptr;        // L2: squared norms, [blocks][256]
    bool borrowed = false;             // device memory belongs to ctx->ds_ws (returned, not freed, by destroy)
};

// device memory of a set: the context's cached workspace when it is free (no cudaMalloc / cudaFree in the steady state), else own allocations
static cudaError_t descset_alloc(sfmb200_descset* s, size_t desc_bytes, size_t exp_bytes, size_t norm_bytes) {
    sfmb200_ctx* ctx = s->ctx;
    if (!ctx->ds_ws.in_use) {
        cudaError_t e = cudaSuccess;
        if (desc_bytes) e = ctx->ds_ws.desc.reserve(desc_bytes);
        if (e == cudaSuccess && exp_bytes) e = ctx->ds_ws.exp.reserve(exp_bytes);
        if (e == cudaSuccess && norm_bytes) e = ctx->ds_ws.norms.reserve(norm_bytes);
        if (e != cudaSuccess) return e;
        ctx->ds_ws.in_use = true; s->borrowed = true;
        s->d_desc = desc_bytes ? (uint32_t*)ctx->ds_ws.desc.p : nullptr;
        s->d_exp = exp_bytes ? (uint8_t*)ctx->ds_ws.exp.p : nullptr;
        s->d_norms = norm_bytes ? (int32_t*)ctx->ds_ws.norms.p : nullptr;
        return cudaSuccess;
    }
    cudaError_t e = cudaSuccess;
    if (desc_bytes) e = cudaMalloc(&s->d_desc, desc_bytes);
    if (e == cudaSuccess && exp_bytes) e = cudaMalloc(&s->d_exp, exp_bytes);
    if (e == cudaSuccess && norm_bytes) e = cudaMalloc(&s->d_norms, norm_bytes);
    return e;
}
static void descset_free(sfmb200_descset* s) {            // caller holds ctx->mu (or is the only user of the set)
    if (s->borrowed) { s->ctx->ds_ws.in_use = false; s->borrowed = false; }
    else { if (s->d_desc) cudaFree(s->d_desc); if (s->d_exp) cudaFree(s->d_exp); if (s->d_norms) cudaFree(s->d_norms); }
    s->d_desc = nullptr; s->d_exp = nullptr; s->d_norms = nullptr;
}

// core: pairs already on the host as PairDesc; descriptors on the device.  Leaves the dense compacted results in
// d_out_* (device) and per-pair dense start positions in d_pair_start [n_pairs+1].
static int match_core(sfmb200_ctx* ctx, const uint32_t* d_desc, const uint8_t* d_exp, int words, const std::vector<PairDesc>& hp, int64_t rows, int nq_max, int nt_max,
                      double ratio, int32_t* d_out_q, int32_t* d_out_t, float* d_out_d, int32_t* d_pair_start, int64_t* d_total, DevBuf& work,
                      int** d_tc_error = nullptr, const int32_t* d_norms = nullptr /* non-null: L2 set */) {
    const bool l2 = d_norms != nullptr;
    const int n_pairs = (int)hp.size();
    const int qblocks = ceil_div(nq_max, QBLOCK);
    // 32-byte descriptors (ORB, the reference's case): exact integer GEMM on the tensor cores (match_tc.cu);
    // SFMB200_MATCH=popc forces the XOR/POPC kernel (other widths always use it)
    const char* mode = getenv("SFMB200_MATCH");
    const bool use_tc = l2 || (words == 8 && d_exp != nullptr && !(mode && strcmp(mode, "popc") == 0));
    const int splits = use_tc ? match_tc_splits(ctx->sm_count, n_pairs, nq_max, nt_max) : choose_splits(ctx->sm_count, (int64_t)qblocks * n_pairs, nt_max);
    const int nblk = (int)ceil_div64(rows, SCAN_THREADS);
    size_t bytes = Carver::pad(sizeof(PairDesc) * n_pairs) + Carver::pad(sizeof(int4) * rows * splits) + Carver::pad(4 * rows) * 3 +
                   Carver::pad(rows) + Carver::pad(4 * (size_t)nblk) + 8192;
    SFM_CUDA(ctx, work.reserve(bytes));
    Carver cv(work.p);
    PairDesc* d_pairs = cv.take<PairDesc>(n_pairs);
    int4* d_partial = cv.take<int4>((size_t)rows * splits);
    int32_t* d_best_t = cv.take<int32_t>(rows); float* d_best_d = cv.take<float>(rows); int32_t* d_rank = cv.take<int32_t>(rows);
    uint8_t* d_flag = cv.take<uint8_t>(rows); int32_t* d_bsum = cv.take<int32_t>(nblk); int* d_err = cv.take<int>(4);
    SFM_CUDA(ctx, cudaMemcpyAsync(d_pairs, hp.data(), sizeof(PairDesc) * n_pairs, cudaMemcpyHostToDevice, ctx->stream));
    dim3 grid(qblocks * splits, n_pairs);
    if (use_tc) {
        SFM_CUDA(ctx, cudaMemsetAsync(d_err, 0, sizeof(int), ctx->stream));
        int rc = match_tc_launch(ctx, l2, d_exp, d_norms, d_pairs, n_pairs, nq_max, splits, d_partial, d_err);
        if (rc) return rc;
        if (d_tc_error) *d_tc_error = d_err;
    } else switch (words) {
        case 4: knn2_hamming_kernel<4><<<grid, KNN_THREADS, 0, ctx->stream>>>(d_desc, d_pairs, qblocks, splits, d_partial); break;
        case 8: knn2_hamming_kernel<8><<<grid, KNN_THREADS, 0, ctx->stream>>>(d_desc, d_pairs, qblocks, splits, d_partial); break;
        case 16: knn2_hamming_kernel<16><<<grid, KNN_THREADS, 0, ctx->stream>>>(d_desc, d_pairs, qblocks, splits, d_partial); break;
        case 32: knn2_hamming_kernel<32><<<grid, KNN_THREADS, 0, ctx->stream>>>(d_desc, d_pairs, qblocks, splits, d_partial); break;
        default: return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "desc_bytes must be 16, 32, 64 or 128 (got %d)", words * 4);
    }
    if (!use_tc) SFM_LAUNCH_CHECK(ctx);
    merge_flag_scan_kernel<<<nblk, SCAN_THREADS, 0, ctx->stream>>>(d_partial, splits, rows, ratio, l2 ? 2 : 0, d_best_t, d_best_d, d_rank, d_flag, d_bsum);
    SFM_LAUNCH_CHECK(ctx);
    scan_sums_kernel<<<1, SCAN_THREADS, 0, ctx->stream>>>(d_bsum, nblk, d_total, use_tc ? d_err : nullptr);
    SFM_LAUNCH_CHECK(ctx);
    scatter_kernel<<<nblk, SCAN_THREADS, 0, ctx->stream>>>(d_pairs, n_pairs, rows, d_best_t, d_best_d, d_rank, d_flag, d_bsum, d_out_q, d_out_t, d_out_d, d_pair_start);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

static int match_pairs_host_out(sfmb200_ctx* ctx, const uint32_t* d_desc, const uint8_t* d_exp, int words, const std::vector<PairDesc>& hp,
                                int64_t rows, int nq_max, int nt_max, double ratio,
                                int32_t* out_q, int32_t* out_t, float* out_d, int64_t* out_off, int32_t* out_cnt, const int32_t* d_norms = nullptr);

static int build_pairs(sfmb200_ctx* ctx, const sfmb200_descset* set, const int32_t* pairs, int n_pairs, std::vector<PairDesc>& hp,
                       int64_t& rows, int& nq_max, int& nt_max) {
    hp.resize(n_pairs); rows = 0; nq_max = 0; nt_max = 0;
    for (int p = 0; p < n_pairs; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        if (l < 0 || r < 0 || l >= set->n_img || r >= set->n_img) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair %d: image id out of range", p);
        PairDesc d; d.q_row = set->img_off[l]; d.nq = set->img_off[l + 1] - d.q_row; d.t_row = set->img_off[r]; d.nt = set->img_off[r + 1] - d.t_row;
        d.out_row = rows; rows += d.nq;
        d.q_blk = set->img_blk.empty() ? 0 : set->img_blk[l]; d.t_blk = set->img_blk.empty() ? 0 : set->img_blk[r];
        hp[p] = d;
        nq_max = std::max(nq_max, d.nq); nt_max = std::max(nt_max, d.nt);
    }
    return SFMB200_OK;
}

static int supported_width(int desc_bytes) {      // the kernels are instantiated for 16/32/64/128 bytes; zero padding keeps every distance
    for (int w : {16, 32, 64, 128}) if (desc_bytes <= w) return w;
    return 0;
}

extern "C" {

int sfmb200_descset_create(sfmb200_ctx* ctx, const uint8_t* desc, const int32_t* img_off, int n_img, int desc_bytes, sfmb200_descset** out) {
    if (!ctx || !out || !img_off || n_img < 0) return SFMB200_ERR_INVALID;
    *out = nullptr;
    const int width = supported_width(desc_bytes);
    if (desc_bytes <= 0 || !width) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "desc_bytes must be in [1, 128] (got %d)", desc_bytes);
    std::vector<uint8_t> padded;                  // widths other than 16/32/64/128 are zero-padded (distances unchanged)
    if (width != desc_bytes && img_off[n_img] > 0) {
        padded.assign((size_t)img_off[n_img] * width, 0);
        for (int64_t r = 0; r < img_off[n_img]; ++r) memcpy(padded.data() + (size_t)r * width, desc + (size_t)r * desc_bytes, desc_bytes);
        desc = padded.data();
    }
    desc_bytes = width;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    sfmb200_descset* s = new sfmb200_descset();
    s->ctx = ctx; s->n_img = n_img; s->words = desc_bytes / 4; s->img_off.assign(img_off, img_off + n_img + 1);
    for (int i = 0; i < n_img; ++i) {
        if (img_off[i + 1] < img_off[i]) { delete s; return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "img_off not monotone"); }
        s->max_rows = std::max(s->max_rows, img_off[i + 1] - img_off[i]);
    }
    const size_t bytes = (size_t)img_off[n_img] * desc_bytes;
    const bool tc = desc_bytes == 32 && img_off[n_img] > 0;      // expanded operand store for the tensor-core kernel
    std::vector<int2> blocks;
    if (tc) {
        const int br = match_tc_block_rows();
        s->img_blk.resize(n_img + 1);
        for (int i = 0; i < n_img; ++i) {
            s->img_blk[i] = (int)blocks.size();
            const int rows = img_off[i + 1] - img_off[i];
            for (int b0 = 0; b0 < rows; b0 += br) blocks.push_back(make_int2(img_off[i] + b0, std::min(br, rows - b0)));
        }
        s->img_blk[n_img] = (int)blocks.size();
    }
    cudaError_t e = descset_alloc(s, bytes + 16, tc ? blocks.size() * match_tc_block_bytes(false) : 0, 0);
    if (e != cudaSuccess) { descset_free(s); delete s; return sfmb200_fail(ctx, SFMB200_ERR_NOMEM, "descriptor set memory (%zu bytes): %s", bytes, cudaGetErrorString(e)); }
    if (bytes) e = cudaMemcpyAsync(s->d_desc, desc, bytes, cudaMemcpyHostToDevice, ctx->stream);
    int rc = SFMB200_OK;
    if (e == cudaSuccess && tc) {
        int2* d_blocks = nullptr;                 // the block list lives in the context's reusable scratch
        e = ctx->scratch2.reserve(Carver::pad(blocks.size() * sizeof(int2) + 16) + 256);
        if (e == cudaSuccess) {
            d_blocks = (int2*)ctx->scratch2.p;
            e = cudaMemcpyAsync(d_blocks, blocks.data(), blocks.size() * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream);
        }
        if (e == cudaSuccess) rc = match_tc_expand(ctx, s->d_desc, d_blocks, (int)blocks.size(), s->d_exp);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);      // the caller's descriptors (and the block list) may go away
    if (e != cudaSuccess || rc) {
        descset_free(s); delete s;
        return sfmb200_fail(ctx, SFMB200_ERR_CUDA, "descriptor upload / operand expansion: %s", cudaGetErrorString(e));
    }
    *out = s;
    return SFMB200_OK;
}

void sfmb200_descset_destroy(sfmb200_descset* s) {
    if (!s) return;
    {
        std::lock_guard<std::mutex> lk(s->ctx->mu);
        cudaSetDevice(s->ctx->device);
        if (s->borrowed) cudaStreamSynchronize(s->ctx->stream);        // nothing of this set may still be in flight when the next set reuses the memory
        descset_free(s);
    }
    delete s;
}

// L2 descriptor set (cv::BFMatcher(NORM_L2) semantics; BASELINE.json configs[3]: SIFT-128): float descriptors [rows][dim], dim <= 128.
// Integer-valued descriptors in [0, 255] (what cv::SIFT produces) are matched EXACTLY on the tensor cores (u8 x u8 -> s32 GEMM,
// match_tc.cu); anything else is refused here (SFMB200_ERR_UNSUPPORTED) -- the per-pair entry point falls back to fp32 SIMT.
int sfmb200_descset_create_l2(sfmb200_ctx* ctx, const float* desc, const int32_t* img_off, int n_img, int dim, sfmb200_descset** out) {
    if (!ctx || !out || !img_off || n_img < 0 || dim <= 0) return SFMB200_ERR_INVALID;
    *out = nullptr;
    if (dim > 128) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "L2 descriptor sets support dim <= 128 (got %d)", dim);
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    sfmb200_descset* s = new sfmb200_descset();
    s->ctx = ctx; s->n_img = n_img; s->words = 32; s->kind = 1; s->img_off.assign(img_off, img_off + n_img + 1);
    const int br = match_tc_block_rows();
    std::vector<int2> blocks;
    s->img_blk.resize(n_img + 1);
    for (int i = 0; i < n_img; ++i) {
        if (img_off[i + 1] < img_off[i]) { delete s; return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "img_off not monotone"); }
        s->max_rows = std::max(s->max_rows, img_off[i + 1] - img_off[i]);
        s->img_blk[i] = (int)blocks.size();
        const int rows = img_off[i + 1] - img_off[i];
        for (int b0 = 0; b0 < rows; b0 += br) blocks.push_back(make_int2(img_off[i] + b0, std::min(br, rows - b0)));
    }
    s->img_blk[n_img] = (int)blocks.size();
    const size_t fbytes = (size_t)img_off[n_img] * dim * sizeof(float), nb = std::max<size_t>(blocks.size(), 1);
    // float staging + block list live in the context's reusable scratch (no cudaMalloc / cudaFree of 100+ MB per set)
    float* d_f = nullptr; int2* d_blocks = nullptr; int* d_bad = nullptr;
    cudaError_t e = ctx->scratch2.reserve(Carver::pad(fbytes + 16) + Carver::pad(nb * sizeof(int2) + 16) + 512);
    if (e == cudaSuccess) {
        Carver cv(ctx->scratch2.p);
        d_f = cv.take<float>((size_t)img_off[n_img] * dim + 4); d_blocks = cv.take<int2>(nb + 2);
        d_bad = reinterpret_cast<int*>(d_blocks + nb);
    }
    if (e == cudaSuccess) e = descset_alloc(s, 0, nb * match_tc_block_bytes(true), nb * br * sizeof(int32_t));
    int h_bad = 0, rc = SFMB200_OK;
    if (e == cudaSuccess && fbytes) e = cudaMemcpyAsync(d_f, desc, fbytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_bad, 0, sizeof(int), ctx->stream);
    if (e == cudaSuccess && !blocks.empty()) {
        e = cudaMemcpyAsync(d_blocks, blocks.data(), blocks.size() * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) rc = match_tc_expand_l2(ctx, d_f, dim, d_blocks, (int)blocks.size(), s->d_exp, s->d_norms, d_bad);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h_bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess || rc || h_bad) {
        descset_free(s);
        delete s;
        if (h_bad) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "L2 descriptor set: values must be integers in [0, 255] (SIFT-like) for the exact tensor-core path");
        return sfmb200_fail(ctx, e == cudaErrorMemoryAllocation ? SFMB200_ERR_NOMEM : SFMB200_ERR_CUDA, "L2 descriptor set: %s", cudaGetErrorString(e));
    }
    *out = s;
    return SFMB200_OK;
}

int sfmb200_match_pairs_device(sfmb200_ctx* ctx, const sfmb200_descset* set, const int32_t* pairs, int n_pairs, double ratio,
                               int32_t* d_out_q, int32_t* d_out_t, float* d_out_d, int32_t* d_pair_start, int64_t* d_total) {
    if (!ctx || !set || (n_pairs > 0 && !pairs) || !d_pair_start || !d_total) return SFMB200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    SFM_CUDA(ctx, cudaMemsetAsync(d_total, 0, sizeof(int64_t), ctx->stream));
    if (n_pairs == 0) return SFMB200_OK;
    SFM_CUDA(ctx, cudaMemsetAsync(d_pair_start, 0, sizeof(int32_t) * n_pairs, ctx->stream));   // pairs without query rows keep 0
    std::vector<PairDesc> hp; int64_t rows; int nq_max, nt_max;
    int rc = build_pairs(ctx, set, pairs, n_pairs, hp, rows, nq_max, nt_max);
    if (rc) return rc;
    if (rows == 0 || nt_max < 2) return SFMB200_OK;
    return match_core(ctx, set->d_desc, set->d_exp, set->words, hp, rows, nq_max, nt_max, ratio, d_out_q, d_out_t, d_out_d, d_pair_start, d_total, ctx->scratch, nullptr, set->d_norms);
}

int sfmb200_match_pairs(sfmb200_ctx* ctx, const sfmb200_descset* set, const int32_t* pairs, int n_pairs, double ratio,
                        int32_t* out_q, int32_t* out_t, float* out_d, int64_t* out_off, int32_t* out_cnt) {
    if (!ctx || !set || n_pairs < 0 || (n_pairs > 0 && (!pairs || !out_off || !out_cnt))) return SFMB200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<PairDesc> hp; int64_t rows; int nq_max, nt_max;
    int rc = build_pairs(ctx, set, pairs, n_pairs, hp, rows, nq_max, nt_max);
    if (rc) return rc;
    return match_pairs_host_out(ctx, set->d_desc, set->d_exp, set->words, hp, rows, nq_max, nt_max, ratio, out_q, out_t, out_d, out_off, out_cnt, set->d_norms);
}

}  // extern "C"

// pairs described on the host, descriptors resident: run the kernels, read back only the survivors.  ctx->mu is held.
static int match_pairs_host_out(sfmb200_ctx* ctx, const uint32_t* d_desc, const uint8_t* d_exp, int words, const std::vector<PairDesc>& hp,
                                int64_t rows, int nq_max, int nt_max, double ratio,
                                int32_t* out_q, int32_t* out_t, float* out_d, int64_t* out_off, int32_t* out_cnt, const int32_t* d_norms) {
    const int n_pairs = (int)hp.size();
    int rc;
    for (int p = 0; p < n_pairs; ++p) { out_off[p] = hp[p].out_row; out_cnt[p] = 0; }
    if (n_pairs) out_off[n_pairs] = rows;
    if (rows == 0) return SFMB200_OK;
    if (nt_max < 2) return SFMB200_OK;   // every pair has < 2 train rows: undefined in the reference -> no matches
    // device outputs (dense) + pair starts + total, behind the kernel workspace
    DevBuf& outb = ctx->scratch;
    DevBuf& dense = ctx->scratch2;       // separate from the kernel workspace, which match_core re-carves
    size_t ob = Carver::pad(4 * rows) * 3 + Carver::pad(4 * (size_t)(n_pairs + 1)) + 512;
    SFM_CUDA(ctx, dense.reserve(ob));
    Carver cv(dense.p);
    int32_t* d_q = cv.take<int32_t>(rows); int32_t* d_t = cv.take<int32_t>(rows); float* d_d = cv.take<float>(rows);
    int32_t* d_start = cv.take<int32_t>(n_pairs + 1); int64_t* d_total = cv.take<int64_t>(1);
    int* d_tc_err = nullptr;
    rc = match_core(ctx, d_desc, d_exp, words, hp, rows, nq_max, nt_max, ratio, d_q, d_t, d_d, d_start, d_total, outb, &d_tc_err, d_norms);
    if (rc) return rc;
    // read back: pair starts + total, then only the survivors
    // (pinned staging is sized for the SURVIVORS, known after the first small read-back -- not for all query rows)
    const size_t head = Carver::pad(sizeof(int32_t) * (n_pairs + 1)) + 512;
    SFM_CUDA(ctx, ctx->pinned.reserve(head));
    int32_t* h_start = (int32_t*)ctx->pinned.p;
    int64_t* h_total = (int64_t*)((char*)ctx->pinned.p + Carver::pad(sizeof(int32_t) * (n_pairs + 1)));
    SFM_CUDA(ctx, cudaMemcpyAsync(h_start, d_start, sizeof(int32_t) * n_pairs, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(h_total, d_total, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    int h_tc_err = 0;
    if (d_tc_err) SFM_CUDA(ctx, cudaMemcpyAsync(&h_tc_err, d_tc_err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h_tc_err) return sfmb200_fail(ctx, SFMB200_ERR_CUDA, "tensor-core matcher: a pipeline barrier timed out");
    const int64_t total = *h_total;
    std::vector<int32_t> starts_copy(h_start, h_start + n_pairs);          // the staging buffer may move when it grows
    SFM_CUDA(ctx, ctx->pinned.reserve(head + 12 * (size_t)total));
    h_start = starts_copy.data();
    char* stage = (char*)ctx->pinned.p + Carver::pad(sizeof(int32_t) * (n_pairs + 1)) + 256;
    int32_t* hq = (int32_t*)stage; int32_t* ht = hq + total; float* hd = (float*)(ht + total);
    if (total) {
        SFM_CUDA(ctx, cudaMemcpyAsync(hq, d_q, 4 * total, cudaMemcpyDeviceToHost, ctx->stream));
        SFM_CUDA(ctx, cudaMemcpyAsync(ht, d_t, 4 * total, cudaMemcpyDeviceToHost, ctx->stream));
        SFM_CUDA(ctx, cudaMemcpyAsync(hd, d_d, 4 * total, cudaMemcpyDeviceToHost, ctx->stream));
        SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    // pairs with zero query rows never wrote their start: fill from the right
    std::vector<int64_t> start(n_pairs + 1);
    start[n_pairs] = total;
    for (int p = n_pairs - 1; p >= 0; --p) start[p] = hp[p].nq > 0 ? h_start[p] : start[p + 1];
    for (int p = 0; p < n_pairs; ++p) {
        const int64_t c = start[p + 1] - start[p];
        out_cnt[p] = (int32_t)c;
        if (c) {
            memcpy(out_q + out_off[p], hq + start[p], 4 * c);
            memcpy(out_t + out_off[p], ht + start[p], 4 * c);
            memcpy(out_d + out_off[p], hd + start[p], 4 * c);
        }
    }
    return SFMB200_OK;
}

// ---- per-call path (what the reference-side shim binds: matchFeatures(const Features&, const Features&)) ------------------
// runSfM() matches every image against every other one (SfM.cpp:166-206), so the per-call entry point sees each image
// N-1 times.  Uploaded (and, for 32-byte descriptors, expanded) images are therefore kept in a context-owned arena keyed
// by (host pointer, rows, width, 64-bit content hash): a pair whose two images are resident costs no cudaMalloc, no
// upload and no expansion.  A hash mismatch (the caller reused a buffer) is a miss; a full arena is flushed whole.
static uint64_t content_hash(const uint8_t* p, size_t n) {
    uint64_t h0 = 0x9E3779B97F4A7C15ull, h1 = 0xC2B2AE3D27D4EB4Full, h2 = 0x165667B19E3779F9ull, h3 = 0x27D4EB2F165667C5ull;
    size_t i = 0;
    for (; i + 32 <= n; i += 32) {
        uint64_t a, b, c, d;
        memcpy(&a, p + i, 8); memcpy(&b, p + i + 8, 8); memcpy(&c, p + i + 16, 8); memcpy(&d, p + i + 24, 8);
        h0 = (h0 ^ a) * 0x100000001B3ull; h0 ^= h0 >> 29;
        h1 = (h1 ^ b) * 0x100000001B3ull; h1 ^= h1 >> 31;
        h2 = (h2 ^ c) * 0x100000001B3ull; h2 ^= h2 >> 27;
        h3 = (h3 ^ d) * 0x100000001B3ull; h3 ^= h3 >> 33;
    }
    for (; i < n; ++i) { h0 = (h0 ^ p[i]) * 0x100000001B3ull; }
    return h0 ^ (h1 * 3) ^ (h2 * 5) ^ (h3 * 7) ^ (uint64_t)n;
}

// make `img` (rows x desc_bytes host bytes) resident; returns its first row / first expanded block in the arena.
// Capacity rule: match_cache_plan keeps rows_cap * width + 16 <= desc.cap and blk_cap * block bytes <= exp.cap after every call,
// recomputing rows_cap from desc.cap whenever the padded width changes (a buffer sized for 16-byte rows holds an eighth as many
// 128-byte rows).  The plan flushes or grows the arena until the call's new images fit under rows_cap / blk_cap; the check below
// holds every placement to the buffers themselves, so a planning mistake is an error status, never a copy past an allocation.
static int cache_acquire(sfmb200_ctx* ctx, const uint8_t* img, int rows, int desc_bytes, int width, uint64_t hash, int& row0, int& blk0) {
    MatchCache& mc = ctx->mcache;
    if (const MatchCacheEntry* e = mc.find(img, rows, desc_bytes, hash)) { row0 = e->row0; blk0 = e->blk0; mc.hits++; return SFMB200_OK; }
    mc.misses++;
    const int br = match_tc_block_rows();
    const int nblk = width == 32 ? ceil_div(rows, br) : 0;
    row0 = (int)mc.rows_used; blk0 = mc.blk_used;
    if (!match_cache_fits(mc, rows, nblk, width, match_tc_block_bytes(false), mc.desc.cap, mc.exp.cap)) {
        const int64_t used = mc.rows_used;
        mc.reset();
        return sfmb200_fail(ctx, SFMB200_ERR_NOMEM, "per-call matcher arena: %d rows of %d bytes at row %lld (+%d blocks at block %d) exceed its "
                            "buffers (%zu / %zu bytes); the arena was cleared", rows, width, (long long)used, nblk, blk0, mc.desc.cap, mc.exp.cap);
    }
    const size_t bytes = (size_t)rows * width;
    if (width == desc_bytes) {
        SFM_CUDA(ctx, cudaMemcpyAsync((char*)mc.desc.p + (size_t)row0 * width, img, bytes, cudaMemcpyHostToDevice, ctx->stream));
    } else {
        std::vector<uint8_t> padded(bytes, 0);
        for (int r = 0; r < rows; ++r) memcpy(padded.data() + (size_t)r * width, img + (size_t)r * desc_bytes, desc_bytes);
        SFM_CUDA(ctx, cudaMemcpyAsync((char*)mc.desc.p + (size_t)row0 * width, padded.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
        SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // `padded` dies with this scope
    }
    if (nblk) {
        std::vector<int2> blocks(nblk);
        for (int b = 0; b < nblk; ++b) blocks[b] = make_int2(row0 + b * br, std::min(br, rows - b * br));
        SFM_CUDA(ctx, ctx->scratch.reserve(sizeof(int2) * nblk + 256));
        SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, blocks.data(), sizeof(int2) * nblk, cudaMemcpyHostToDevice, ctx->stream));
        int rc = match_tc_expand(ctx, (const uint32_t*)mc.desc.p, (const int2*)ctx->scratch.p, nblk, (uint8_t*)mc.exp.p + (size_t)blk0 * match_tc_block_bytes(false));
        if (rc) return rc;
    }
    mc.rows_used += rows; mc.blk_used += nblk;
    mc.entries.push_back({img, rows, desc_bytes, hash, row0, blk0});
    return SFMB200_OK;
}

extern "C" {

int sfmb200_match_knn2_ratio(sfmb200_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int desc_bytes,
                             double ratio, int32_t* out_q, int32_t* out_t, float* out_d, int* out_n) {
    if (!ctx || !out_n || nq < 0 || nt < 0) return SFMB200_ERR_INVALID;
    *out_n = 0;
    if (nq == 0 || nt < 2) return SFMB200_OK;     // nt < 2: undefined behaviour in the reference (:65) -> empty
    if (!q || !t || !out_q || !out_t || !out_d) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    const int width = supported_width(desc_bytes);
    if (desc_bytes <= 0 || !width) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "desc_bytes must be in [1, 128] (got %d)", desc_bytes);
    const uint64_t hq = content_hash(q, (size_t)nq * desc_bytes), ht = content_hash(t, (size_t)nt * desc_bytes);   // outside the lock
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    MatchCache& mc = ctx->mcache;
    const char* env = getenv("SFMB200_MATCH_CACHE");
    const bool keep = !(env && env[0] == '0');
    const MatchCachePlan plan = match_cache_plan(mc, mc.desc.cap, width, keep, desc_bytes, q, nq, hq, t, nt, ht, match_tc_block_rows(),
                                                 match_tc_block_bytes(false));
    if (plan.desc_bytes || plan.exp_bytes) {
        SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        cudaError_t e = plan.desc_bytes ? mc.desc.reserve(plan.desc_bytes) : cudaSuccess;
        if (e == cudaSuccess && plan.exp_bytes) e = mc.exp.reserve(plan.exp_bytes);
        if (e != cudaSuccess) mc.reset();
        SFM_CUDA(ctx, e);
    }
    PairDesc pd; pd.out_row = 0; pd.nq = nq; pd.nt = nt;
    int rc = cache_acquire(ctx, q, nq, desc_bytes, width, hq, pd.q_row, pd.q_blk);
    if (rc) return rc;
    rc = cache_acquire(ctx, t, nt, desc_bytes, width, ht, pd.t_row, pd.t_blk);
    if (rc) return rc;
    std::vector<PairDesc> hp(1, pd);
    int64_t ooff[2]; int32_t cnt[1];
    rc = match_pairs_host_out(ctx, (const uint32_t*)mc.desc.p, width == 32 ? (const uint8_t*)mc.exp.p : nullptr, width / 4, hp, nq, nq, nt, ratio,
                              out_q, out_t, out_d, ooff, cnt);
    if (rc) { mc.flush(); return rc; }
    *out_n = cnt[0];
    return SFMB200_OK;
}

int sfmb200_match_knn2_ratio_l2(sfmb200_ctx* ctx, const float* q, int nq, const float* t, int nt, int dim,
                                double ratio, int32_t* out_q, int32_t* out_t, float* out_d, int* out_n) {
    if (!ctx || !out_n || nq < 0 || nt < 0 || dim <= 0) return SFMB200_ERR_INVALID;
    *out_n = 0;
    if (nq == 0 || nt < 2) return SFMB200_OK;
    if (!q || !t || !out_q || !out_t || !out_d) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (dim <= 128 && !(getenv("SFMB200_MATCH_L2") && strcmp(getenv("SFMB200_MATCH_L2"), "simt") == 0)) {
        // exact integer GEMM on the tensor cores when the descriptors are u8-valued (SIFT): a two-image descriptor set
        std::vector<float> both((size_t)(nq + nt) * dim);
        memcpy(both.data(), q, sizeof(float) * (size_t)nq * dim);
        memcpy(both.data() + (size_t)nq * dim, t, sizeof(float) * (size_t)nt * dim);
        const int32_t off[3] = {0, nq, nq + nt};
        sfmb200_descset* set = nullptr;
        int rc = sfmb200_descset_create_l2(ctx, both.data(), off, 2, dim, &set);
        if (rc == SFMB200_OK) {
            const int32_t pair[2] = {0, 1};
            int64_t ooff[2]; int32_t cnt[1];
            rc = sfmb200_match_pairs(ctx, set, pair, 1, ratio, out_q, out_t, out_d, ooff, cnt);
            sfmb200_descset_destroy(set);
            if (rc) return rc;
            *out_n = cnt[0];
            return SFMB200_OK;
        }
        if (rc != SFMB200_ERR_UNSUPPORTED) return rc;          // not u8-valued: fp32 SIMT kernel below
    }
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const int64_t rows = nq;
    int splits = 1;
    while ((int64_t)nq * splits < 8LL * ctx->sm_count * 8 && splits < 32 && nt / (splits * 2) >= 64) splits *= 2;
    const int nblk = (int)ceil_div64(rows, SCAN_THREADS);
    size_t bytes = Carver::pad(4 * (size_t)nq * dim) + Carver::pad(4 * (size_t)nt * dim) + Carver::pad(sizeof(PairDesc)) +
                   Carver::pad(16 * rows * splits) + Carver::pad(4 * rows) * 6 + Carver::pad(rows) + Carver::pad(4 * (size_t)nblk) + 4096;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    float* d_qf = cv.take<float>((size_t)nq * dim); float* d_tf = cv.take<float>((size_t)nt * dim);
    PairDesc* d_pairs = cv.take<PairDesc>(1); float4* d_partial = cv.take<float4>((size_t)rows * splits);
    int32_t* d_best_t = cv.take<int32_t>(rows); float* d_best_d = cv.take<float>(rows); int32_t* d_rank = cv.take<int32_t>(rows);
    int32_t* d_q = cv.take<int32_t>(rows); int32_t* d_t = cv.take<int32_t>(rows); float* d_d = cv.take<float>(rows);
    uint8_t* d_flag = cv.take<uint8_t>(rows); int32_t* d_bsum = cv.take<int32_t>(nblk);
    int32_t* d_start = cv.take<int32_t>(2); int64_t* d_total = cv.take<int64_t>(1);
    PairDesc hp = {0, nq, 0, nt, 0};
    SFM_CUDA(ctx, cudaMemcpyAsync(d_qf, q, 4 * (size_t)nq * dim, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_tf, t, 4 * (size_t)nt * dim, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_pairs, &hp, sizeof hp, cudaMemcpyHostToDevice, ctx->stream));
    const int64_t warps = (int64_t)nq * splits;
    knn2_l2_kernel<<<(unsigned)ceil_div64(warps * 32, 256), 256, 0, ctx->stream>>>(d_qf, nq, d_tf, nt, dim, splits, d_partial);
    SFM_LAUNCH_CHECK(ctx);
    merge_flag_scan_kernel<<<nblk, SCAN_THREADS, 0, ctx->stream>>>((const int4*)d_partial, splits, rows, ratio, 1, d_best_t, d_best_d, d_rank, d_flag, d_bsum);
    SFM_LAUNCH_CHECK(ctx);
    scan_sums_kernel<<<1, SCAN_THREADS, 0, ctx->stream>>>(d_bsum, nblk, d_total, nullptr);
    SFM_LAUNCH_CHECK(ctx);
    scatter_kernel<<<nblk, SCAN_THREADS, 0, ctx->stream>>>(d_pairs, 1, rows, d_best_t, d_best_d, d_rank, d_flag, d_bsum, d_q, d_t, d_d, d_start);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, ctx->pinned.reserve(64 + 12 * (size_t)rows));
    int64_t* h_total = (int64_t*)ctx->pinned.p;
    SFM_CUDA(ctx, cudaMemcpyAsync(h_total, d_total, 8, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int64_t total = *h_total;
    if (total) {
        SFM_CUDA(ctx, cudaMemcpyAsync(out_q, d_q, 4 * total, cudaMemcpyDeviceToHost, ctx->stream));
        SFM_CUDA(ctx, cudaMemcpyAsync(out_t, d_t, 4 * total, cudaMemcpyDeviceToHost, ctx->stream));
        SFM_CUDA(ctx, cudaMemcpyAsync(out_d, d_d, 4 * total, cudaMemcpyDeviceToHost, ctx->stream));
        SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    *out_n = (int)total;
    return SFMB200_OK;
}

}  // extern "C"
