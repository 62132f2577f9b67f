// essential.cu -- K5: essential-matrix RANSAC and pose recovery for a batch of image pairs on the device (SURVEY.md 8 row f-2).
//
// Replaces SfMStereoUtilities::findCameraMatricesFromMatch (reference SfMToyLib/SfMStereoUtilities.cpp:74-118):
//   cv::findEssentialMat(RANSAC, 0.999, 1 px) -> cv::recoverPose(E, ..., mask)
// for every pair of a call (sfmb200_find_camera_matrices_pairs; sfmb200_find_camera_matrices is a call with one pair).  The
// correspondences of all pairs are concatenated; pair p draws S_p samples (0 for m < 5, 1 for m == 5, else max_iters).  The pairs
// are cut into consecutive groups whose hypotheses (10 slots of 96 B per sample) fit ES_HYP_BUDGET; per group, three launches
// (four with the OpenCV sampler):
//   0. essential_cv_sample_kernel  SFMB200_SAMPLER_OPENCV only, one thread per pair of the group: the pair's S samples as
//                                  cv::findEssentialMat draws them (em_cv_samples: cv::RNG((uint64)-1), getSubset's redraws),
//                                  serially, since a redraw shifts the rest of the stream
//   1. essential_solve_kernel      one thread per sample of the group: its 5 distinct correspondences (drawn here with
//                                  splitmix64 keyed by seed, the sample's index within its pair and draw, or read from launch
//                                  0), normalised, five-point solver (essential_math.cuh) -> up to 10 E per sample in slot 10 s + k
//   2. essential_score_kernel      one CTA per sample: every point of the pair is normalised once and tested against all the
//                                  sample's solutions with the Sampson error and inlier rule of is_inlier<1> (ransac_score.cuh,
//                                  the arithmetic sfmb200_ransac_score pins against cv2); empty slots score 0
//   3. essential_select_kernel     one warp per pair: the warp stages 32 samples' counts at a time, lane 0 replays OpenCV's
//                                  sequential loop (RANSACPointSetRegistrator::run) over them in (sample, solution) order, then
//                                  decomposeEssentialMat of the winner
// and once over the concatenated matches of all pairs, each CTA covering 128 matches of one pair:
//   4. essential_cheirality_kernel the inlier mask of the winner (is_inlier<1>), DLT triangulation (dlt_math.cuh,
//                                  cv::triangulatePoints' algorithm) against the four pose candidates, recoverPose's depth tests,
//                                  per-pair, per-candidate counts
//   5. essential_pose_kernel       per pair the first candidate with the largest count (recoverPose's if-chain): R, t, pruning mask
// One upload, one download, one host synchronisation per call.  A pair's outputs depend on its own matches and the options only:
// not on the other pairs of the call, its position or the grouping.
// For a call with one pair the samples, solution counts and per-slot inlier counts stay on the device (ctx->ess_trace) for
// sfmb200_essential_last_trace.
#include <algorithm>

#include "ransac_score.cuh"
#include "dlt_math.cuh"
#include "essential_math.cuh"

namespace {

constexpr int ES_SOLVE_THREADS = 32;     // one sample per thread; 1000 samples of one pair spread over 32 SMs
constexpr int ES_SCORE_THREADS = 128;    // one sample per CTA; the pairs of a run have a few hundred to a few thousand matches
constexpr int ES_SELECT_WARPS = 4;       // one pair per warp
constexpr int ES_POINT_THREADS = 128;
constexpr int ES_CV_SAMPLE_THREADS = 32;  // one pair per thread; a group holds a few hundred pairs at max_iters 1000
constexpr size_t ES_HYP_BUDGET = size_t(256) << 20;    // device bytes of hypotheses per group of pairs

struct EsPair {
    int64_t off;        // first match of the pair in the concatenated arrays
    int32_t m;          // matches
    int32_t S;          // samples drawn
    int32_t s0;         // first sample of the pair in its group
    int32_t b0;         // first CTA of the pair in the cheirality and pose launches
};

struct EssResult {
    double E[9], R[9], t[3];
    int32_t n_inliers, n_good, iterations, n_hypotheses, found, pad;
};

// The pair of pr[0..np) that owns sample / CTA `key`: the last one whose first sample / CTA (field F) is <= key.  A pair without
// samples or CTAs starts where the next one does, so the search passes over it.
template <int32_t EsPair::*F>
__device__ __forceinline__ int es_owner(const EsPair* __restrict__ pr, int np, int key) {
    int lo = 0, hi = np - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (pr[mid].*F <= key) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// one thread per pair of the group: the pair's samples as cv::findEssentialMat draws them (em_cv_samples), into the group's buffer
__global__ void __launch_bounds__(ES_CV_SAMPLE_THREADS)
essential_cv_sample_kernel(const EsPair* __restrict__ pr, int np, int32_t* __restrict__ samples) {
    const int p = blockIdx.x * ES_CV_SAMPLE_THREADS + threadIdx.x;
    if (p >= np) return;
    const EsPair P = pr[p];
    em_cv_samples(P.m, P.S, samples + 5 * (size_t)P.s0);
}

__global__ void __launch_bounds__(ES_SOLVE_THREADS)
essential_solve_kernel(const float* __restrict__ ga, const float* __restrict__ gb, const EsPair* __restrict__ pr, int np, int Sg, uint64_t seed,
                       bool drawn, double f, double cx, double cy, int32_t* __restrict__ samples, int32_t* __restrict__ nsol, Model* __restrict__ hyp) {
    const int s = blockIdx.x * ES_SOLVE_THREADS + threadIdx.x;
    if (s >= Sg) return;
    const EsPair P = pr[es_owner<&EsPair::s0>(pr, np, s)];
    const float* a = ga + 2 * P.off;
    const float* b = gb + 2 * P.off;
    int idx[5];
    if (drawn) {
#pragma unroll
        for (int j = 0; j < 5; ++j) idx[j] = samples[5 * s + j];
    } else {
        em_sample(seed, (uint32_t)(s - P.s0), P.m, idx);
    }
    double x1[5][2], x2[5][2];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        // cv::findEssentialMat(points, focal, pp): (x - cx) / focal in double, the normalisation is_inlier<1> applies
        x1[j][0] = ((double)a[2 * idx[j]] - cx) / f; x1[j][1] = ((double)a[2 * idx[j] + 1] - cy) / f;
        x2[j][0] = ((double)b[2 * idx[j]] - cx) / f; x2[j][1] = ((double)b[2 * idx[j] + 1] - cy) / f;
        if (!drawn) samples[5 * s + j] = idx[j];
    }
    double E[10][9];
    const int c = five_point_solve(x1, x2, E);
    nsol[s] = c;
    for (int k = 0; k < c; ++k) {
        Model& M = hyp[10 * (size_t)s + k];
#pragma unroll
        for (int q = 0; q < 9; ++q) M.m[q] = E[k][q];
        M.m[9] = M.m[10] = M.m[11] = 0.0;
    }
}

__global__ void __launch_bounds__(ES_SOLVE_THREADS)
five_point_kernel(const double* __restrict__ x1, const double* __restrict__ x2, int ns, double* __restrict__ E, int32_t* __restrict__ nsol) {
    const int s = blockIdx.x * ES_SOLVE_THREADS + threadIdx.x;
    if (s >= ns) return;
    double a[5][2], b[5][2], e[10][9];
    for (int j = 0; j < 10; ++j) { a[j >> 1][j & 1] = x1[10 * (size_t)s + j]; b[j >> 1][j & 1] = x2[10 * (size_t)s + j]; }
    const int c = five_point_solve(a, b, e);
    nsol[s] = c;
    for (int k = 0; k < 10; ++k)
        for (int q = 0; q < 9; ++q) E[90 * (size_t)s + 9 * k + q] = k < c ? e[k][q] : 0.0;
}

// one CTA per sample: each point of the pair is normalised once, as is_inlier<1> normalises it, and tested against every solution of
// the sample; a CTA owns its counts, so they are deterministic without atomics
__global__ void __launch_bounds__(ES_SCORE_THREADS)
essential_score_kernel(const float* __restrict__ ga, const float* __restrict__ gb, const EsPair* __restrict__ pr, int np, const Model* __restrict__ hyp,
                       const int32_t* __restrict__ nsol, double f, double cx, double cy, float t2, int32_t* __restrict__ counts) {
    constexpr int W = ES_SCORE_THREADS / 32;
    __shared__ double M[10][9];
    __shared__ int wsum[W][10];
    const int s = blockIdx.x;
    const int c = nsol[s];
    for (int q = threadIdx.x; q < 9 * c; q += ES_SCORE_THREADS) M[q / 9][q % 9] = hyp[10 * (size_t)s + q / 9].m[q % 9];
    __syncthreads();
    const EsPair P = pr[es_owner<&EsPair::s0>(pr, np, s)];
    const float* a = ga + 2 * P.off;
    const float* b = gb + 2 * P.off;
    int cnt[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) cnt[k] = 0;
    for (int i = threadIdx.x; c > 0 && i < P.m; i += ES_SCORE_THREADS) {
        const double x1 = ((double)a[2 * i] - cx) / f, y1 = ((double)a[2 * i + 1] - cy) / f;
        const double x2 = ((double)b[2 * i] - cx) / f, y2 = ((double)b[2 * i + 1] - cy) / f;
#pragma unroll
        for (int k = 0; k < 10; ++k)
            if (k < c) cnt[k] += err_essential(M[k], x1, y1, x2, y2) <= t2 ? 1 : 0;
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) {
        int v = cnt[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 10) {
        int v = 0;
        for (int w = 0; w < W; ++w) v += wsum[w][threadIdx.x];
        counts[10 * (size_t)s + threadIdx.x] = v;
    }
}

__global__ void __launch_bounds__(32 * ES_SELECT_WARPS)
essential_select_kernel(const EsPair* __restrict__ pr, int np, const int32_t* __restrict__ nsol, const int32_t* __restrict__ counts, const Model* __restrict__ hyp,
                        int max_iters, double confidence, EssResult* __restrict__ res, double* __restrict__ cand, int32_t* __restrict__ cnt4) {
    __shared__ int32_t sn[ES_SELECT_WARPS][32], sc[ES_SELECT_WARPS][320];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int p = blockIdx.x * ES_SELECT_WARPS + w;
    if (p >= np) return;
    const EsPair P = pr[p];
    const int32_t* ns = nsol + P.s0;
    const int32_t* cs = counts + 10 * (size_t)P.s0;
    SeqSelect st;
    seq_select_begin(st, max_iters);
    int nh = 0;
    for (int base = 0; base < P.S; base += 32) {
        const int k = min(32, P.S - base);
        const int v = lane < k ? ns[base + lane] : 0;
        nh += v;
        if (!__shfl_sync(0xffffffffu, st.iter < st.niters, 0)) continue;    // the loop has stopped: only the solution total is left
        sn[w][lane] = v;
        for (int q = lane; q < 10 * k; q += 32) sc[w][q] = cs[10 * (size_t)base + q];
        __syncwarp();
        if (lane == 0) seq_select_chunk(st, sn[w], sc[w], 10, k, P.m, confidence, 5, 10 * P.s0);
        __syncwarp();
    }
    const int best = st.best, max_good = st.max_good, iter = st.iter;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nh += __shfl_xor_sync(0xffffffffu, nh, o);
    if (lane != 0) return;
    EssResult& r = res[p];
    double* cp = cand + 48 * (size_t)p;
    for (int c = 0; c < 4; ++c) cnt4[4 * p + c] = 0;
    r.iterations = iter; r.n_hypotheses = nh; r.n_good = 0;
    double R1[9], R2[9], t[3];
    const bool ok = best >= 0 && em_decompose_essential(hyp[best].m, R1, R2, t);
    r.found = ok ? 1 : 0;
    r.n_inliers = ok ? max_good : 0;
    for (int q = 0; q < 9; ++q) { r.E[q] = ok ? hyp[best].m[q] : 0.0; r.R[q] = 0.0; }
    r.t[0] = r.t[1] = r.t[2] = 0.0;
    if (!ok) return;
    // candidates in recoverPose's order: [R1|t], [R2|t], [R1|-t], [R2|-t]
    for (int c = 0; c < 4; ++c)
        for (int row = 0; row < 3; ++row) {
            const double* Rc = (c & 1) ? R2 : R1;
            for (int q = 0; q < 3; ++q) cp[12 * c + 4 * row + q] = Rc[3 * row + q];
            cp[12 * c + 4 * row + 3] = (c & 2) ? -t[row] : t[row];
        }
}

// launched with ES_POINT_THREADS; a register limit instead of __launch_bounds__, under which ptxas stops at 128 registers and spills
__global__ void __maxnreg__(168)
essential_cheirality_kernel(const float* __restrict__ ga, const float* __restrict__ gb, const EsPair* __restrict__ pr, int np, double f, double cx, double cy,
                            float t2, const EssResult* __restrict__ res, const double* __restrict__ cand, double dist, uint8_t* __restrict__ inl,
                            uint8_t* __restrict__ bits, int32_t* __restrict__ cnt4) {
    const int p = es_owner<&EsPair::b0>(pr, np, blockIdx.x);
    const EsPair P = pr[p];
    const int i = (blockIdx.x - P.b0) * ES_POINT_THREADS + threadIdx.x;
    const float* a = ga + 2 * P.off;
    const float* b = gb + 2 * P.off;
    bool in = false;
    unsigned bm = 0;
    if (i < P.m && res[p].found) {
        // the inlier test of is_inlier<1> on the point it normalises
        const double x1 = ((double)a[2 * i] - cx) / f, y1 = ((double)a[2 * i + 1] - cy) / f;
        const double x2 = ((double)b[2 * i] - cx) / f, y2 = ((double)b[2 * i + 1] - cy) / f;
        in = err_essential(res[p].E, x1, y1, x2, y2) <= t2;
        for (int c = 0; in && c < 4; ++c) {
            const double* Pc = cand + 48 * (size_t)p + 12 * c;
            // cv::triangulatePoints rows x P[2] - P[0], y P[2] - P[1] for P0 = [I|0] and P
            double A[4][4] = {{-1.0, 0.0, x1, 0.0}, {0.0, -1.0, y1, 0.0}, {0, 0, 0, 0}, {0, 0, 0, 0}}, Q[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) { A[2][k] = x2 * Pc[8 + k] - Pc[k]; A[3][k] = y2 * Pc[8 + k] - Pc[4 + k]; }
            if (!null_vector_fast(A, Q)) null_vector_4x4(A, Q);
            // recoverPose: Q2 Q3 > 0, Q /= Q3, depth < dist in the first camera, 0 < (P Q).z < dist in the second
            bool ok = Q[2] * Q[3] > 0.0;
            const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3];
            ok = ok && Z < dist;
            const double z2 = Pc[8] * X + Pc[9] * Y + Pc[10] * Z + Pc[11];
            ok = ok && z2 > 0.0 && z2 < dist;
            bm |= (ok ? 1u : 0u) << c;
        }
    }
    if (i < P.m) { inl[P.off + i] = in ? 1 : 0; bits[P.off + i] = (uint8_t)bm; }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const unsigned v = __ballot_sync(0xffffffffu, (bm >> c) & 1u);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(cnt4 + 4 * p + c, __popc(v));
    }
}

__global__ void __launch_bounds__(ES_POINT_THREADS)
essential_pose_kernel(const EsPair* __restrict__ pr, int np, const uint8_t* __restrict__ bits, const int32_t* __restrict__ cnt4, const double* __restrict__ cand,
                      EssResult* __restrict__ res, uint8_t* __restrict__ pose_mask) {
    const int p = es_owner<&EsPair::b0>(pr, np, blockIdx.x);
    const EsPair P = pr[p];
    const int i = (blockIdx.x - P.b0) * ES_POINT_THREADS + threadIdx.x;
    const int g0 = cnt4[4 * p], g1 = cnt4[4 * p + 1], g2 = cnt4[4 * p + 2], g3 = cnt4[4 * p + 3];
    const int c = (g0 >= g1 && g0 >= g2 && g0 >= g3) ? 0 : (g1 >= g0 && g1 >= g2 && g1 >= g3) ? 1 : (g2 >= g0 && g2 >= g1 && g2 >= g3) ? 2 : 3;
    if (i < P.m) pose_mask[P.off + i] = (bits[P.off + i] >> c) & 1;
    if (i == 0 && res[p].found) {
        const double* cp = cand + 48 * (size_t)p;
        for (int r = 0; r < 3; ++r) {
            for (int q = 0; q < 3; ++q) res[p].R[3 * r + q] = cp[12 * c + 4 * r + q];
            res[p].t[r] = cp[12 * c + 4 * r + 3];
        }
        res[p].n_good = c == 0 ? g0 : c == 1 ? g1 : c == 2 ? g2 : g3;
    }
}

int es_check_options(sfmb200_ctx* ctx, const sfmb200_essential_options& o) {
    if (o.max_iters < 1 || !(o.confidence > 0.0 && o.confidence < 1.0) || !(o.threshold_px > 0.0) || !(o.distance_thresh > 0.0))
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "essential options: max_iters >= 1, confidence in (0, 1), threshold_px > 0, distance_thresh > 0");
    if ((size_t)o.max_iters * 10 > (size_t)INT32_MAX / 2) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "max_iters too large");
    if (o.sampler != SFMB200_SAMPLER_SEEDED && o.sampler != SFMB200_SAMPLER_OPENCV)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "essential options: sampler must be SFMB200_SAMPLER_SEEDED or SFMB200_SAMPLER_OPENCV");
    return SFMB200_OK;
}

// The launches of one call over n_pairs pairs: pair p owns matches moff[p] .. moff[p+1] of the concatenated left / right pixel
// coordinates that gather(a, b) writes into the pinned staging.  Outputs were zeroed by the caller; those of a pair with a model
// are filled here, summary for every pair.
template <class Gather>
int es_run(sfmb200_ctx* ctx, const sfmb200_essential_options& o, double focal, double cx, double cy, int n_pairs, const int64_t* moff,
           Gather gather, double* E, double* R, double* t, uint8_t* inlier_mask, uint8_t* pose_mask, sfmb200_essential_summary* summary) {
    const int64_t M = moff[n_pairs];
    // consecutive pairs form a group while their hypotheses fit the budget; a pair that alone exceeds it is a group of its own
    const size_t group_cap = ES_HYP_BUDGET / (10 * sizeof(Model));
    std::vector<EsPair> pr(n_pairs);
    std::vector<int> groups{0};
    size_t gs = 0, smax = 0;
    int nb = 0;
    for (int p = 0; p < n_pairs; ++p) {
        const int m = (int)(moff[p + 1] - moff[p]);
        const int S = m < 5 ? 0 : m == 5 ? 1 : o.max_iters;      // five correspondences: every sample would hold the same five points
        if (gs > 0 && gs + S > group_cap) { groups.push_back(p); gs = 0; }
        pr[p] = EsPair{moff[p], m, S, (int32_t)gs, nb};
        gs += S; smax = std::max(smax, gs);
        nb += ceil_div(m, ES_POINT_THREADS);
    }
    groups.push_back(n_pairs);
    const size_t slots = 10 * smax;

    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    // pinned staging: pairs | a | b on the way in; results | inlier masks | pose masks on the way out.  The device carving has the
    // same layout, so each direction is one copy.
    const size_t in_bytes = Carver::pad(sizeof(EsPair) * n_pairs) + 2 * Carver::pad(8 * (size_t)M);
    const size_t out_bytes = Carver::pad(sizeof(EssResult) * n_pairs) + 2 * Carver::pad((size_t)M);
    SFM_CUDA(ctx, ctx->pinned.reserve(in_bytes + out_bytes + 256));
    Carver hc(ctx->pinned.p);
    EsPair* h_pr = hc.take<EsPair>(n_pairs);
    float* h_a = hc.take<float>(2 * (size_t)M);
    float* h_b = hc.take<float>(2 * (size_t)M);
    EssResult* h_res = hc.take<EssResult>(n_pairs);
    uint8_t* h_inl = hc.take<uint8_t>((size_t)M);
    uint8_t* h_pose = hc.take<uint8_t>((size_t)M);
    const size_t in_len = (char*)h_b + 8 * (size_t)M - (char*)ctx->pinned.p;
    const size_t out_off = (char*)h_res - (char*)ctx->pinned.p, out_len = hc.off - out_off;
    memcpy(h_pr, pr.data(), sizeof(EsPair) * n_pairs);
    gather(h_a, h_b);

    const size_t bytes = in_bytes + out_bytes + Carver::pad((size_t)M) + Carver::pad(48 * 8 * (size_t)n_pairs) + Carver::pad(16 * (size_t)n_pairs) +
                         Carver::pad(sizeof(Model) * slots) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    const EsPair* d_pr = cv.take<EsPair>(n_pairs);
    const float* d_a = cv.take<float>(2 * (size_t)M);
    const float* d_b = cv.take<float>(2 * (size_t)M);
    EssResult* d_res = cv.take<EssResult>(n_pairs);
    uint8_t* d_inl = cv.take<uint8_t>((size_t)M);
    uint8_t* d_pose = cv.take<uint8_t>((size_t)M);
    uint8_t* d_bits = cv.take<uint8_t>((size_t)M);
    double* d_cand = cv.take<double>(48 * (size_t)n_pairs);
    int32_t* d_cnt4 = cv.take<int32_t>(4 * (size_t)n_pairs);
    Model* d_hyp = cv.take<Model>(slots);
    SFM_CUDA(ctx, ctx->ess_trace.reserve(Carver::pad(4 * 5 * smax) + Carver::pad(4 * smax) + Carver::pad(4 * slots) + 1024));
    Carver tc(ctx->ess_trace.p);
    int32_t* d_samples = tc.take<int32_t>(5 * smax);
    int32_t* d_nsol = tc.take<int32_t>(smax);
    int32_t* d_counts = tc.take<int32_t>(slots);
    ctx->ess_trace_samples = 0;

    SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, ctx->pinned.p, in_len, cudaMemcpyHostToDevice, ctx->stream));
    const float t2 = (float)((o.threshold_px / focal) * (o.threshold_px / focal));      // findEssentialMat: threshold /= focal
    for (size_t g = 0; g + 1 < groups.size(); ++g) {
        const int p0 = groups[g], np = groups[g + 1] - p0;
        const int Sg = pr[p0 + np - 1].s0 + pr[p0 + np - 1].S;
        if (Sg > 0) {
            const bool drawn = o.sampler == SFMB200_SAMPLER_OPENCV;
            if (drawn) {
                essential_cv_sample_kernel<<<ceil_div(np, ES_CV_SAMPLE_THREADS), ES_CV_SAMPLE_THREADS, 0, ctx->stream>>>(d_pr + p0, np, d_samples);
                SFM_LAUNCH_CHECK(ctx);
            }
            essential_solve_kernel<<<ceil_div(Sg, ES_SOLVE_THREADS), ES_SOLVE_THREADS, 0, ctx->stream>>>(d_a, d_b, d_pr + p0, np, Sg, o.seed, drawn, focal,
                                                                                                         cx, cy, d_samples, d_nsol, d_hyp);
            SFM_LAUNCH_CHECK(ctx);
            essential_score_kernel<<<Sg, ES_SCORE_THREADS, 0, ctx->stream>>>(d_a, d_b, d_pr + p0, np, d_hyp, d_nsol, focal, cx, cy, t2, d_counts);
            SFM_LAUNCH_CHECK(ctx);
        }
        essential_select_kernel<<<ceil_div(np, ES_SELECT_WARPS), 32 * ES_SELECT_WARPS, 0, ctx->stream>>>(
            d_pr + p0, np, d_nsol, d_counts, d_hyp, o.max_iters, o.confidence, d_res + p0, d_cand + 48 * (size_t)p0, d_cnt4 + 4 * (size_t)p0);
        SFM_LAUNCH_CHECK(ctx);
    }
    if (nb > 0) {
        essential_cheirality_kernel<<<nb, ES_POINT_THREADS, 0, ctx->stream>>>(d_a, d_b, d_pr, n_pairs, focal, cx, cy, t2, d_res, d_cand, o.distance_thresh,
                                                                            d_inl, d_bits, d_cnt4);
        SFM_LAUNCH_CHECK(ctx);
        essential_pose_kernel<<<nb, ES_POINT_THREADS, 0, ctx->stream>>>(d_pr, n_pairs, d_bits, d_cnt4, d_cand, d_res, d_pose);
        SFM_LAUNCH_CHECK(ctx);
    }
    SFM_CUDA(ctx, cudaMemcpyAsync((char*)ctx->pinned.p + out_off, (char*)ctx->scratch.p + out_off, out_len, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->ess_trace_samples = n_pairs == 1 ? pr[0].S : 0;

    for (int p = 0; p < n_pairs; ++p) {
        const EssResult& r = h_res[p];
        if (summary) {
            sfmb200_essential_summary& sm = summary[p];
            sm.found = r.found; sm.n_inliers = r.n_inliers; sm.n_good = r.n_good; sm.iterations = r.iterations;
            sm.n_samples = pr[p].S; sm.n_hypotheses = r.n_hypotheses;
        }
        if (!r.found) continue;
        if (E) memcpy(E + 9 * (size_t)p, r.E, 9 * sizeof(double));
        if (R) memcpy(R + 9 * (size_t)p, r.R, 9 * sizeof(double));
        if (t) memcpy(t + 3 * (size_t)p, r.t, 3 * sizeof(double));
        if (inlier_mask) memcpy(inlier_mask + moff[p], h_inl + moff[p], (size_t)pr[p].m);
        if (pose_mask) memcpy(pose_mask + moff[p], h_pose + moff[p], (size_t)pr[p].m);
    }
    return SFMB200_OK;
}

}  // namespace

extern "C" {

void sfmb200_essential_default_options(sfmb200_essential_options* opt) {
    if (!opt) return;
    opt->max_iters = 1000; opt->confidence = 0.999; opt->threshold_px = 1.0; opt->distance_thresh = 50.0; opt->seed = 0;
    opt->sampler = SFMB200_SAMPLER_SEEDED;
}

int sfmb200_find_camera_matrices(sfmb200_ctx* ctx, const float* K, const float* pts_left, int n_left, const float* pts_right, int n_right,
                                 const int32_t* match_q, const int32_t* match_t, int m, const sfmb200_essential_options* opt,
                                 double* E, double* R, double* t, uint8_t* inlier_mask, uint8_t* pose_mask, sfmb200_essential_summary* summary) {
    if (!ctx || !K || m < 0 || n_left < 0 || n_right < 0) return SFMB200_ERR_INVALID;
    sfmb200_essential_options o;
    sfmb200_essential_default_options(&o);
    if (opt) o = *opt;
    if (const int rc = es_check_options(ctx, o)) return rc;
    const double focal = (double)K[0], cx = (double)K[2], cy = (double)K[5];
    if (!(focal != 0.0) || !std::isfinite(focal) || !std::isfinite(cx) || !std::isfinite(cy)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "K: focal length must be finite and nonzero");
    if (summary) memset(summary, 0, sizeof(sfmb200_essential_summary));
    if (E) memset(E, 0, 9 * sizeof(double));
    if (R) memset(R, 0, 9 * sizeof(double));
    if (t) memset(t, 0, 3 * sizeof(double));
    if (inlier_mask) memset(inlier_mask, 0, (size_t)m);
    if (pose_mask) memset(pose_mask, 0, (size_t)m);
    if (m > 0 && (!pts_left || !pts_right)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (const int rc = check_two_view_matches(ctx, match_q, match_t, m, n_left, n_right)) return rc;
    if (m < 5) return SFMB200_OK;
    const int64_t moff[2] = {0, m};
    return es_run(ctx, o, focal, cx, cy, 1, moff, [&](float* ha, float* hb) {
        for (int i = 0; i < m; ++i) {
            const int iq = match_q ? match_q[i] : i, it = match_t ? match_t[i] : i;
            ha[2 * i] = pts_left[2 * (size_t)iq]; ha[2 * i + 1] = pts_left[2 * (size_t)iq + 1];
            hb[2 * i] = pts_right[2 * (size_t)it]; hb[2 * i + 1] = pts_right[2 * (size_t)it + 1];
        }
    }, E, R, t, inlier_mask, pose_mask, summary);
}

int sfmb200_find_camera_matrices_pairs(sfmb200_ctx* ctx, const float* K, const float* pts, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs,
                                       const int32_t* match_q, const int32_t* match_t, const int64_t* match_off, const sfmb200_essential_options* opt,
                                       double* E, double* R, double* t, uint8_t* inlier_mask, uint8_t* pose_mask, sfmb200_essential_summary* summary) {
    if (!ctx || n_img < 0 || n_pairs < 0) return SFMB200_ERR_INVALID;
    sfmb200_essential_options o;
    sfmb200_essential_default_options(&o);
    if (opt) o = *opt;
    if (const int rc = es_check_options(ctx, o)) return rc;
    if (!K) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    const double focal = (double)K[0], cx = (double)K[2], cy = (double)K[5];
    if (!(focal != 0.0) || !std::isfinite(focal) || !std::isfinite(cx) || !std::isfinite(cy)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "K: focal length must be finite and nonzero");
    if (n_pairs == 0) return SFMB200_OK;
    int64_t M = 0;
    if (const int rc = check_pair_batch(ctx, pts, img_off, n_img, pairs, n_pairs, match_q, match_t, match_off, INT32_MAX / 2, &M)) return rc;
    if (summary) memset(summary, 0, sizeof(sfmb200_essential_summary) * (size_t)n_pairs);
    if (E) memset(E, 0, 9 * sizeof(double) * (size_t)n_pairs);
    if (R) memset(R, 0, 9 * sizeof(double) * (size_t)n_pairs);
    if (t) memset(t, 0, 3 * sizeof(double) * (size_t)n_pairs);
    if (inlier_mask) memset(inlier_mask, 0, (size_t)M);
    if (pose_mask) memset(pose_mask, 0, (size_t)M);
    return es_run(ctx, o, focal, cx, cy, n_pairs, match_off, [&](float* ha, float* hb) {
        for (int p = 0; p < n_pairs; ++p) {
            const float* L = pts + 2 * (size_t)img_off[pairs[2 * p]];
            const float* Rt = pts + 2 * (size_t)img_off[pairs[2 * p + 1]];
            for (int64_t k = match_off[p]; k < match_off[p + 1]; ++k) {
                ha[2 * k] = L[2 * (size_t)match_q[k]]; ha[2 * k + 1] = L[2 * (size_t)match_q[k] + 1];
                hb[2 * k] = Rt[2 * (size_t)match_t[k]]; hb[2 * k + 1] = Rt[2 * (size_t)match_t[k] + 1];
            }
        }
    }, E, R, t, inlier_mask, pose_mask, summary);
}

int sfmb200_five_point(sfmb200_ctx* ctx, const double* x1, const double* x2, int ns, double* E, int32_t* nsol) {
    if (!ctx || ns < 0) return SFMB200_ERR_INVALID;
    if (ns == 0) return SFMB200_OK;
    if (!x1 || !x2 || !E || !nsol) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t bytes = 2 * Carver::pad(80 * (size_t)ns) + Carver::pad(720 * (size_t)ns) + Carver::pad(4 * (size_t)ns) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    double* d_x1 = cv.take<double>(10 * (size_t)ns); double* d_x2 = cv.take<double>(10 * (size_t)ns);
    double* d_E = cv.take<double>(90 * (size_t)ns); int32_t* d_n = cv.take<int32_t>(ns);
    SFM_CUDA(ctx, cudaMemcpyAsync(d_x1, x1, 80 * (size_t)ns, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_x2, x2, 80 * (size_t)ns, cudaMemcpyHostToDevice, ctx->stream));
    five_point_kernel<<<ceil_div(ns, ES_SOLVE_THREADS), ES_SOLVE_THREADS, 0, ctx->stream>>>(d_x1, d_x2, ns, d_E, d_n);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaMemcpyAsync(E, d_E, 720 * (size_t)ns, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(nsol, d_n, 4 * (size_t)ns, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SFMB200_OK;
}

int sfmb200_essential_last_trace(sfmb200_ctx* ctx, int cap, int32_t* samples, int32_t* nsol, int32_t* counts) {
    if (!ctx || cap < 0) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    const int S = ctx->ess_trace_samples;
    const int k = cap < S ? cap : S;
    if (k == 0) return S;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
    Carver tc(ctx->ess_trace.p);
    int32_t* d_samples = tc.take<int32_t>(5 * (size_t)S);
    int32_t* d_nsol = tc.take<int32_t>(S);
    int32_t* d_counts = tc.take<int32_t>(10 * (size_t)S);
    std::vector<int32_t> hn(k), hc(10 * (size_t)k);
    if (samples && cudaMemcpyAsync(samples, d_samples, 20 * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (cudaMemcpyAsync(hn.data(), d_nsol, 4 * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (cudaMemcpyAsync(hc.data(), d_counts, 40 * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return -1;
    if (nsol) memcpy(nsol, hn.data(), 4 * (size_t)k);
    if (counts) {                            // slots 10 s + j, j < nsol[s], compacted in (sample, solution) order
        size_t o = 0;
        for (int s = 0; s < k; ++s)
            for (int j = 0; j < hn[s]; ++j) counts[o++] = hc[10 * (size_t)s + j];
    }
    return S;
}

}  // extern "C"
