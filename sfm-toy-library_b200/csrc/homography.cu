// homography.cu -- K6: homography RANSAC for a batch of image pairs on the device (SURVEY.md 8 row f-2).
//
// Replaces SfMStereoUtilities::findHomographyInliers (reference SfMToyLib/SfMStereoUtilities.cpp:51-72), which
// SfM::sortViewsForBaseline calls once per image pair:  cv::findHomography(RANSAC, 10 px) -> countNonZero(mask).
// One launch, one CTA per pair, one host synchronisation per call.  Inside a CTA:
//   0. the pair's correspondences are gathered from the key points of its two images into a contiguous scratch;
//   1. thread 0 draws the next HG_BATCH quads with cv::RNG and getSubset (serial: a rejected quad shifts the stream);
//   2. one thread per quad solves the normalised 4-point DLT (homography_math.cuh);
//   3. the CTA scores the batch against all correspondences with is_inlier<0> (ransac_score.cuh, the arithmetic
//      sfmb200_ransac_score pins against cv2); integer counts, so the reduction order does not matter;
//   4. thread 0 replays OpenCV's sequential selection over the batch; quads drawn beyond the sample budget are discarded,
//      so the speculation never changes the result;
//   5. after the loop: the DLT on the best model's inliers (three block reductions: coordinate sums, deviation sums, L^T L),
//      Levenberg-Marquardt on h00..h21 (a block reduction of J^T J, J^T r, r.r per evaluation, the 8 x 8 solve on thread 0),
//      and the final mask of the refined H.
// The floating-point block reductions run in a fixed order for a fixed block size, so outputs are bitwise reproducible and do not
// depend on which other pairs share the call.
#include "ransac_score.cuh"
#include "homography_math.cuh"

namespace {

constexpr int HG_THREADS = 128;
constexpr int HG_WARPS = HG_THREADS / 32;
constexpr int HG_BATCH = 32;           // quads drawn, solved and scored per round; the crazyhorse pairs visit 4-130

struct HgOut {
    double H[9];
    int32_t found, n_inliers, ransac_inliers, iterations;
};

struct HgShared {
    double Hq[HG_BATCH][9];
    int32_t quad[HG_BATCH][4];
    int32_t ok[HG_BATCH], cnt[HG_BATCH];
    double bestH[9], Hr[9];
    double red[HG_WARPS][HM_LM_TERMS + 1];
    double acc[HM_LM_TERMS + 1];
    HmNorm nm;
    HmLm lm;
    uint64_t rng;
    int32_t nb, fail, iter, niters, max_good, stop, flag, n_final;
};

// sum over the CTA of K per-thread values (the last one reduced with max when LAST_MAX); the result lands in out[0..K) for all
// threads.  Fixed order: a shuffle tree inside each warp, then the warps in index order on thread 0.
template <int K, bool LAST_MAX>
__device__ __forceinline__ void hg_block_reduce(double* v, HgShared& s, double* out) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double x = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double y = __shfl_xor_sync(0xffffffffu, x, o);
            x = (LAST_MAX && k == K - 1) ? fmax(x, y) : x + y;
        }
        if (lane == 0) s.red[w][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        const int k = threadIdx.x;
        double x = s.red[0][k];
        for (int q = 1; q < HG_WARPS; ++q) x = (LAST_MAX && k == K - 1) ? fmax(x, s.red[q][k]) : x + s.red[q][k];
        out[k] = x;
    }
    __syncthreads();
}

__device__ __forceinline__ bool hg_inlier(const double* H, const float* a, const float* b, int i, float t2) {
    return is_inlier<0>(H, nullptr, a, b, i, t2);
}

// J^T J, J^T r, r.r and max |r| at h over the inliers of the RANSAC model -> s.acc
__device__ void hg_lm_eval(const double* h, const float* a, const float* b, int n, float t2, HgShared& s) {
    double v[HM_LM_TERMS + 1];
#pragma unroll
    for (int k = 0; k <= HM_LM_TERMS; ++k) v[k] = 0.0;
    for (int i = threadIdx.x; i < n; i += HG_THREADS)
        if (hg_inlier(s.bestH, a, b, i, t2)) hm_lm_add(h, a[2 * i], a[2 * i + 1], b[2 * i], b[2 * i + 1], v, v[HM_LM_TERMS]);
    hg_block_reduce<HM_LM_TERMS + 1, true>(v, s, s.acc);
}

__global__ void __launch_bounds__(HG_THREADS)
homography_pairs_kernel(const float* __restrict__ pts, const int32_t* __restrict__ img_off, const int32_t* __restrict__ pairs,
                        const int32_t* __restrict__ mq, const int32_t* __restrict__ mt, const int64_t* __restrict__ moff,
                        int max_iters, double confidence, float t2, int refine_iters, float* __restrict__ ga, float* __restrict__ gb,
                        HgOut* __restrict__ out, uint8_t* __restrict__ mask, int32_t* __restrict__ tr_quad, int32_t* __restrict__ tr_cnt) {
    __shared__ HgShared s;
    const int p = blockIdx.x, tid = threadIdx.x;
    const int64_t o = moff[p];
    const int n = (int)(moff[p + 1] - o);
    const float* P0 = pts + 2 * (size_t)img_off[pairs[2 * p]];
    const float* P1 = pts + 2 * (size_t)img_off[pairs[2 * p + 1]];
    float* a = ga + 2 * o;
    float* b = gb + 2 * o;
    uint8_t* pm = mask + o;
    for (int i = tid; i < n; i += HG_THREADS) {
        const int q = mq[o + i], t = mt[o + i];
        a[2 * i] = P0[2 * q]; a[2 * i + 1] = P0[2 * q + 1];
        b[2 * i] = P1[2 * t]; b[2 * i + 1] = P1[2 * t + 1];
    }
    __syncthreads();
    HgOut& r = out[p];

    if (n <= 4) {                     // findHomography: fewer than 4 points -> no model; exactly 4 -> their DLT, mask all ones
        if (tid == 0) {
            double H[9];
            const bool ok = n == 4 && hm_kernel(a, b, 4, H);
            for (int k = 0; k < 9; ++k) r.H[k] = ok ? H[k] : 0.0;
            r.found = ok; r.n_inliers = r.ransac_inliers = ok ? 4 : 0; r.iterations = 0;
            s.flag = ok;
        }
        __syncthreads();
        for (int i = tid; i < n; i += HG_THREADS) pm[i] = (uint8_t)s.flag;
        return;
    }

    // ---- RANSAC: speculative batches, sequential selection ----
    if (tid == 0) { s.rng = ~0ull; s.iter = 0; s.niters = max(max_iters, 1); s.max_good = 0; s.stop = 0; }
    __syncthreads();
    while (true) {
        if (tid == 0) {
            const int want = min(HG_BATCH, s.niters - s.iter);
            int nb = 0;
            s.fail = 0;
            for (; nb < want; ++nb)
                if (!hm_draw_subset(s.rng, n, a, b, s.quad[nb])) { s.fail = 1; break; }
            s.nb = nb;
        }
        __syncthreads();
        const int nb = s.nb;
        if (tid < nb) {
            float qa[8], qb[8];
            for (int j = 0; j < 4; ++j) {
                const int v = s.quad[tid][j];
                qa[2 * j] = a[2 * v]; qa[2 * j + 1] = a[2 * v + 1]; qb[2 * j] = b[2 * v]; qb[2 * j + 1] = b[2 * v + 1];
            }
            s.ok[tid] = hm_kernel(qa, qb, 4, s.Hq[tid]) ? 1 : 0;
            s.cnt[tid] = 0;
        }
        __syncthreads();
        int c[HG_BATCH];
#pragma unroll
        for (int k = 0; k < HG_BATCH; ++k) c[k] = 0;
        for (int i = tid; i < n; i += HG_THREADS) {
#pragma unroll
            for (int k = 0; k < HG_BATCH; ++k)
                if (k < nb && s.ok[k]) c[k] += hg_inlier(s.Hq[k], a, b, i, t2) ? 1 : 0;
        }
#pragma unroll
        for (int k = 0; k < HG_BATCH; ++k) {
            if (k >= nb) break;
            int x = c[k];
#pragma unroll
            for (int q = 16; q > 0; q >>= 1) x += __shfl_xor_sync(0xffffffffu, x, q);
            if ((tid & 31) == 0 && x) atomicAdd(&s.cnt[k], x);
        }
        __syncthreads();
        if (tid == 0) {
            for (int k = 0; k < nb && s.iter < s.niters; ++k) {
                const int g = s.ok[k] ? s.cnt[k] : -1;
                if (tr_quad) {
                    const size_t slot = (size_t)p * max_iters + s.iter;
                    for (int j = 0; j < 4; ++j) tr_quad[4 * slot + j] = s.quad[k][j];
                    tr_cnt[slot] = g;
                }
                if (g > max(s.max_good, 3)) {
                    for (int q = 0; q < 9; ++q) s.bestH[q] = s.Hq[k][q];
                    s.max_good = g;
                    s.niters = ransac_update_num_iters(confidence, (double)(n - g) / n, 4, s.niters);
                }
                ++s.iter;
            }
            s.stop = s.fail || s.iter >= s.niters;     // getSubset gave up: no model at the first sample, otherwise the loop ends
        }
        __syncthreads();
        if (s.stop) break;
    }
    if (s.max_good == 0) {
        if (tid == 0) {
            for (int k = 0; k < 9; ++k) r.H[k] = 0.0;
            r.found = 0; r.n_inliers = r.ransac_inliers = 0; r.iterations = s.iter;
        }
        for (int i = tid; i < n; i += HG_THREADS) pm[i] = 0;
        return;
    }

    // ---- refit: the DLT on the RANSAC inliers ----
    {
        double v[4] = {0, 0, 0, 0};
        for (int i = tid; i < n; i += HG_THREADS)
            if (hg_inlier(s.bestH, a, b, i, t2)) { v[0] += a[2 * i]; v[1] += a[2 * i + 1]; v[2] += b[2 * i]; v[3] += b[2 * i + 1]; }
        hg_block_reduce<4, false>(v, s, s.acc);
        if (tid == 0) {
            const int cnt = s.max_good;
            s.nm.cMx = s.acc[0] / cnt; s.nm.cMy = s.acc[1] / cnt; s.nm.cmx = s.acc[2] / cnt; s.nm.cmy = s.acc[3] / cnt;
        }
        __syncthreads();
        v[0] = v[1] = v[2] = v[3] = 0.0;
        for (int i = tid; i < n; i += HG_THREADS)
            if (hg_inlier(s.bestH, a, b, i, t2)) {
                v[0] += fabs(a[2 * i] - s.nm.cMx); v[1] += fabs(a[2 * i + 1] - s.nm.cMy);
                v[2] += fabs(b[2 * i] - s.nm.cmx); v[3] += fabs(b[2 * i + 1] - s.nm.cmy);
            }
        hg_block_reduce<4, false>(v, s, s.acc);
        if (tid == 0) s.flag = hm_norm_finish(s.max_good, s.acc, s.nm) ? 1 : 0;
        __syncthreads();
        if (s.flag) {
            double L[45];
#pragma unroll
            for (int k = 0; k < 45; ++k) L[k] = 0.0;
            for (int i = tid; i < n; i += HG_THREADS)
                if (hg_inlier(s.bestH, a, b, i, t2)) hm_ltl_add(s.nm, a[2 * i], a[2 * i + 1], b[2 * i], b[2 * i + 1], L);
            hg_block_reduce<45, false>(L, s, s.acc);
        }
        if (tid == 0) {
            if (s.flag) hm_solve_ltl(s.acc, s.nm, s.Hr);
            else for (int k = 0; k < 9; ++k) s.Hr[k] = s.bestH[k];      // runKernel failed: findHomography keeps the RANSAC model
        }
        __syncthreads();
    }

    // ---- Levenberg-Marquardt on h00..h21 ----
    hg_lm_eval(s.Hr, a, b, n, t2, s);
    if (tid == 0) hm_lm_init(s.lm, s.Hr, s.acc, s.acc[HM_LM_TERMS]);
    __syncthreads();
    for (;;) {
        if (tid == 0) hm_lm_propose(s.lm);
        __syncthreads();
        double sd = 0.0;
        for (int i = tid; i < n; i += HG_THREADS)
            if (hg_inlier(s.bestH, a, b, i, t2)) {
                double rr[2];
                hm_residual(s.lm.xd, a[2 * i], a[2 * i + 1], b[2 * i], b[2 * i + 1], rr, nullptr);
                sd += rr[0] * rr[0] + rr[1] * rr[1];
            }
        hg_block_reduce<1, false>(&sd, s, s.acc);
        if (tid == 0) s.flag = hm_lm_update(s.lm, s.acc[0]) ? 1 : 0;
        __syncthreads();
        if (s.flag) {
            hg_lm_eval(s.lm.x, a, b, n, t2, s);
            if (tid == 0) hm_lm_load(s.lm, s.acc, s.acc[HM_LM_TERMS]);
        }
        if (tid == 0) s.stop = hm_lm_proceed(s.lm, refine_iters) ? 0 : 1;
        __syncthreads();
        if (s.stop) break;
    }
    if (tid == 0) {
        for (int k = 0; k < 8; ++k) s.Hr[k] = s.lm.x[k];
        s.Hr[8] = 1.0;
        s.n_final = 0;
    }
    __syncthreads();

    // ---- the returned mask: inliers of the refined H ----
    int cnt = 0;
    for (int i = tid; i < n; i += HG_THREADS) {
        const bool in = hg_inlier(s.Hr, a, b, i, t2);
        pm[i] = in ? 1 : 0;
        cnt += in ? 1 : 0;
    }
#pragma unroll
    for (int q = 16; q > 0; q >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, q);
    if ((tid & 31) == 0 && cnt) atomicAdd(&s.n_final, cnt);
    __syncthreads();
    if (tid == 0) {
        for (int k = 0; k < 9; ++k) r.H[k] = s.Hr[k];
        r.found = 1; r.n_inliers = s.n_final; r.ransac_inliers = s.max_good; r.iterations = s.iter;
    }
}

}  // namespace

extern "C" {

void sfmb200_homography_default_options(sfmb200_homography_options* opt) {
    if (!opt) return;
    opt->max_iters = 2000; opt->confidence = 0.995; opt->threshold_px = 10.0; opt->refine_iters = 10; opt->record_trace = 0;
}

int sfmb200_find_homography_pairs(sfmb200_ctx* ctx, const float* pts, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs,
                                  const int32_t* match_q, const int32_t* match_t, const int64_t* match_off,
                                  const sfmb200_homography_options* opt, double* H, uint8_t* mask, sfmb200_homography_summary* summary) {
    if (!ctx || n_img < 0 || n_pairs < 0) return SFMB200_ERR_INVALID;
    sfmb200_homography_options o;
    sfmb200_homography_default_options(&o);
    if (opt) o = *opt;
    if (o.max_iters < 1 || !(o.confidence > 0.0 && o.confidence < 1.0) || !(o.threshold_px > 0.0) || o.refine_iters < 1 ||
        (o.record_trace != 0 && o.record_trace != 1))
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "homography options: max_iters >= 1, confidence in (0, 1), threshold_px > 0, refine_iters >= 1, record_trace 0 or 1");
    if (!img_off || (n_pairs > 0 && (!pairs || !match_off))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (img_off[0] != 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "img_off[0] must be 0");
    for (int i = 0; i < n_img; ++i)
        if (img_off[i + 1] < img_off[i]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "img_off is not monotone at image %d", i);
    const int64_t n_pts = img_off[n_img];
    if (n_pts > 0 && !pts) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (n_pairs > 0 && match_off[0] != 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_off[0] must be 0");
    for (int p = 0; p < n_pairs; ++p) {
        if (match_off[p + 1] < match_off[p]) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_off is not monotone at pair %d", p);
        if (pairs[2 * p] < 0 || pairs[2 * p] >= n_img || pairs[2 * p + 1] < 0 || pairs[2 * p + 1] >= n_img)
            return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pair %d names an image outside [0, %d)", p, n_img);
    }
    const int64_t M = n_pairs > 0 ? match_off[n_pairs] : 0;
    if (M > INT32_MAX / 2) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "too many matches in one call");
    if (M > 0 && (!match_q || !match_t)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    for (int p = 0; p < n_pairs; ++p) {
        const int nl = img_off[pairs[2 * p] + 1] - img_off[pairs[2 * p]], nr = img_off[pairs[2 * p + 1] + 1] - img_off[pairs[2 * p + 1]];
        for (int64_t k = match_off[p]; k < match_off[p + 1]; ++k)
            if (match_q[k] < 0 || match_q[k] >= nl || match_t[k] < 0 || match_t[k] >= nr)
                return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match %lld of pair %d indexes outside its images' key points", (long long)k, p);
    }
    if ((size_t)n_pairs * (size_t)o.max_iters > (size_t)INT32_MAX / 4 && o.record_trace)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "trace too large: n_pairs * max_iters");
    if (summary) memset(summary, 0, sizeof(sfmb200_homography_summary) * (size_t)n_pairs);
    if (H) memset(H, 0, 9 * sizeof(double) * (size_t)n_pairs);
    if (mask) memset(mask, 0, (size_t)M);
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->hg_trace_pairs = 0;
    ctx->hg_trace_visited.clear();
    if (n_pairs == 0) return SFMB200_OK;
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));

    // pinned staging: pts | img_off | pairs | match_off | match_q | match_t on the way in; results | mask on the way out
    const size_t b_pts = 8 * (size_t)n_pts, b_off = 4 * ((size_t)n_img + 1), b_pairs = 8 * (size_t)n_pairs, b_moff = 8 * ((size_t)n_pairs + 1),
                 b_m = 4 * (size_t)M;
    const size_t in_bytes = Carver::pad(b_pts) + Carver::pad(b_off) + Carver::pad(b_pairs) + Carver::pad(b_moff) + 2 * Carver::pad(b_m);
    const size_t out_bytes = Carver::pad(sizeof(HgOut) * (size_t)n_pairs) + Carver::pad((size_t)M);
    SFM_CUDA(ctx, ctx->pinned.reserve(in_bytes + out_bytes + 256));
    Carver hc(ctx->pinned.p);
    float* h_pts = hc.take<float>(2 * (size_t)n_pts);
    int32_t* h_off = hc.take<int32_t>((size_t)n_img + 1);
    int32_t* h_pairs = hc.take<int32_t>(2 * (size_t)n_pairs);
    int64_t* h_moff = hc.take<int64_t>((size_t)n_pairs + 1);
    int32_t* h_mq = hc.take<int32_t>((size_t)M);
    int32_t* h_mt = hc.take<int32_t>((size_t)M);
    HgOut* h_out = hc.take<HgOut>(n_pairs);
    uint8_t* h_mask = hc.take<uint8_t>((size_t)M);
    if (n_pts) memcpy(h_pts, pts, b_pts);
    memcpy(h_off, img_off, b_off); memcpy(h_pairs, pairs, b_pairs); memcpy(h_moff, match_off, b_moff);
    if (M) { memcpy(h_mq, match_q, b_m); memcpy(h_mt, match_t, b_m); }

    const size_t bytes = in_bytes + 2 * Carver::pad(8 * (size_t)M) + Carver::pad(sizeof(HgOut) * (size_t)n_pairs) + Carver::pad((size_t)M) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    char* d_in = (char*)ctx->scratch.p;
    const float* d_pts = cv.take<float>(2 * (size_t)n_pts);
    const int32_t* d_off = cv.take<int32_t>((size_t)n_img + 1);
    const int32_t* d_pairs = cv.take<int32_t>(2 * (size_t)n_pairs);
    const int64_t* d_moff = cv.take<int64_t>((size_t)n_pairs + 1);
    const int32_t* d_mq = cv.take<int32_t>((size_t)M);
    const int32_t* d_mt = cv.take<int32_t>((size_t)M);
    float* d_a = cv.take<float>(2 * (size_t)M);
    float* d_b = cv.take<float>(2 * (size_t)M);
    HgOut* d_out = cv.take<HgOut>(n_pairs);
    uint8_t* d_mask = cv.take<uint8_t>((size_t)M);
    int32_t *d_tq = nullptr, *d_tc = nullptr;
    if (o.record_trace) {
        const size_t slots = (size_t)n_pairs * o.max_iters;
        SFM_CUDA(ctx, ctx->hg_trace.reserve(Carver::pad(16 * slots) + Carver::pad(4 * slots) + 512));
        Carver tc(ctx->hg_trace.p);
        d_tq = tc.take<int32_t>(4 * slots);
        d_tc = tc.take<int32_t>(slots);
    }

    // the host and device carvings have the same layout, so the whole input goes in one copy
    SFM_CUDA(ctx, cudaMemcpyAsync(d_in, ctx->pinned.p, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    const float t2 = (float)(o.threshold_px * o.threshold_px);
    homography_pairs_kernel<<<n_pairs, HG_THREADS, 0, ctx->stream>>>(d_pts, d_off, d_pairs, d_mq, d_mt, d_moff, o.max_iters, o.confidence, t2,
                                                                      o.refine_iters, d_a, d_b, d_out, d_mask, d_tq, d_tc);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaMemcpyAsync(h_out, d_out, sizeof(HgOut) * (size_t)n_pairs, cudaMemcpyDeviceToHost, ctx->stream));
    if (M) SFM_CUDA(ctx, cudaMemcpyAsync(h_mask, d_mask, (size_t)M, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

    if (o.record_trace) {
        ctx->hg_trace_pairs = n_pairs; ctx->hg_trace_stride = o.max_iters;
        ctx->hg_trace_visited.resize(n_pairs);
    }
    for (int p = 0; p < n_pairs; ++p) {
        const HgOut& r = h_out[p];
        if (summary) { summary[p].found = r.found; summary[p].n_inliers = r.n_inliers; summary[p].ransac_inliers = r.ransac_inliers; summary[p].iterations = r.iterations; }
        if (H && r.found) memcpy(H + 9 * (size_t)p, r.H, 9 * sizeof(double));
        if (o.record_trace) ctx->hg_trace_visited[p] = r.iterations;
    }
    if (mask && M) memcpy(mask, h_mask, (size_t)M);
    return SFMB200_OK;
}

int sfmb200_homography_last_trace(sfmb200_ctx* ctx, int pair, int cap, int32_t* quads, int32_t* counts) {
    if (!ctx || cap < 0) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (pair < 0 || pair >= ctx->hg_trace_pairs) return -1;
    const int v = ctx->hg_trace_visited[pair];
    const int k = cap < v ? cap : v;
    if (k == 0) return v;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
    const size_t slots = (size_t)ctx->hg_trace_pairs * ctx->hg_trace_stride, base = (size_t)pair * ctx->hg_trace_stride;
    Carver tc(ctx->hg_trace.p);
    const int32_t* d_tq = tc.take<int32_t>(4 * slots);
    const int32_t* d_tc = tc.take<int32_t>(slots);
    if (quads && cudaMemcpyAsync(quads, d_tq + 4 * base, 16 * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (counts && cudaMemcpyAsync(counts, d_tc + base, 4 * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return -1;
    return v;
}

}  // extern "C"
