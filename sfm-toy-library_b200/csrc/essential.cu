// essential.cu -- K5: essential-matrix RANSAC and pose recovery on the device (SURVEY.md 8 row f-2).
//
// Replaces SfMStereoUtilities::findCameraMatricesFromMatch (reference SfMToyLib/SfMStereoUtilities.cpp:74-118):
//   cv::findEssentialMat(RANSAC, 0.999, 1 px) -> cv::recoverPose(E, ..., mask)
// One call, seven launches, one host synchronisation:
//   1. essential_solve_kernel      one thread per sample: draw 5 distinct correspondences (splitmix64 keyed by seed, sample
//                                  and draw), normalise them, five-point solver (essential_math.cuh) -> up to 10 E per sample
//                                  in slot 10 s + k
//   2. essential_score_kernel      one CTA per slot: inliers of the solution with is_inlier<1> (ransac_score.cuh, the
//                                  arithmetic sfmb200_ransac_score pins against cv2); empty slots score 0
//   3. essential_select_kernel     one thread: OpenCV's sequential loop (RANSACPointSetRegistrator::run) replayed over the
//                                  counts in (sample, solution) order, then decomposeEssentialMat of the winner
//   4. ransac_mask_kernel<1>       the inlier mask of the winner (ransac_score.cuh)
//   5. essential_cheirality_kernel one thread per point: DLT triangulation (dlt_math.cuh, cv::triangulatePoints' algorithm)
//                                  against the four pose candidates, recoverPose's depth tests, per-candidate counts
//   6. essential_pose_kernel       the first candidate with the largest count (recoverPose's if-chain): R, t, pruning mask
// The samples, solution counts and per-slot inlier counts stay on the device (ctx->ess_trace) for
// sfmb200_essential_last_trace.
#include "ransac_score.cuh"
#include "dlt_math.cuh"
#include "essential_math.cuh"

namespace {

constexpr int ES_SOLVE_THREADS = 32;     // one sample per thread; 1000 samples spread over 32 SMs
constexpr int ES_POINT_THREADS = 128;

struct EssResult {
    double E[9], R[9], t[3];
    int32_t best_slot;      // slot of the winner, -1 = none (read by ransac_mask_kernel as best[0])
    int32_t n_inliers, n_good, iterations, n_hypotheses, found;
};

__global__ void __launch_bounds__(ES_SOLVE_THREADS)
essential_solve_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, int S, uint64_t seed, double f, double cx, double cy,
                       int32_t* __restrict__ samples, int32_t* __restrict__ nsol, Model* __restrict__ hyp) {
    const int s = blockIdx.x * ES_SOLVE_THREADS + threadIdx.x;
    if (s >= S) return;
    int idx[5];
    em_sample(seed, (uint32_t)s, n, idx);
    double x1[5][2], x2[5][2];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        // cv::findEssentialMat(points, focal, pp): (x - cx) / focal in double, the normalisation is_inlier<1> applies
        x1[j][0] = ((double)a[2 * idx[j]] - cx) / f; x1[j][1] = ((double)a[2 * idx[j] + 1] - cy) / f;
        x2[j][0] = ((double)b[2 * idx[j]] - cx) / f; x2[j][1] = ((double)b[2 * idx[j] + 1] - cy) / f;
        samples[5 * s + j] = idx[j];
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

// one CTA per slot; a CTA owns its whole count, so the counts are deterministic without atomics
__global__ void __launch_bounds__(RS_THREADS)
essential_score_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, const Model* __restrict__ hyp, const int32_t* __restrict__ nsol,
                       const double* __restrict__ aux, float t2, int32_t* __restrict__ counts) {
    const int h = blockIdx.x;
    if (h % 10 >= nsol[h / 10]) {
        if (threadIdx.x == 0) counts[h] = 0;
        return;
    }
    __shared__ double M[12], A[9];
    __shared__ int wsum[RS_THREADS / 32];
    if (threadIdx.x < 12) M[threadIdx.x] = hyp[h].m[threadIdx.x];
    if (threadIdx.x < 9) A[threadIdx.x] = aux[threadIdx.x];
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < n; i += RS_THREADS) c += is_inlier<1>(M, A, a, b, i, t2) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < RS_THREADS / 32; ++w) s += wsum[w];
        counts[h] = s;
    }
}

__global__ void __launch_bounds__(32)
essential_select_kernel(const int32_t* __restrict__ nsol, const int32_t* __restrict__ counts, const Model* __restrict__ hyp, int S, int n,
                        int max_iters, double confidence, EssResult* __restrict__ res, double* __restrict__ cand, int32_t* __restrict__ cnt4) {
    if (threadIdx.x != 0) return;
    int niters = max(max_iters, 1), best = -1, max_good = 0, iter = 0, nh = 0;
    for (; iter < niters && iter < S; ++iter)
        for (int k = 0; k < nsol[iter]; ++k) {
            const int g = counts[10 * iter + k];
            if (g > max(max_good, 4)) {
                best = 10 * iter + k; max_good = g;
                niters = ransac_update_num_iters(confidence, (double)(n - g) / n, 5, niters);
            }
        }
    for (int s = 0; s < S; ++s) nh += nsol[s];
    for (int c = 0; c < 4; ++c) cnt4[c] = 0;
    res->iterations = iter; res->n_hypotheses = nh; res->n_good = 0;
    double R1[9], R2[9], t[3];
    const bool ok = best >= 0 && em_decompose_essential(hyp[best].m, R1, R2, t);
    res->found = ok ? 1 : 0;
    res->best_slot = ok ? best : -1;
    res->n_inliers = ok ? max_good : 0;
    for (int q = 0; q < 9; ++q) { res->E[q] = ok ? hyp[best].m[q] : 0.0; res->R[q] = 0.0; }
    res->t[0] = res->t[1] = res->t[2] = 0.0;
    if (!ok) return;
    // candidates in recoverPose's order: [R1|t], [R2|t], [R1|-t], [R2|-t]
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 3; ++r) {
            const double* R = (c & 1) ? R2 : R1;
            for (int q = 0; q < 3; ++q) cand[12 * c + 4 * r + q] = R[3 * r + q];
            cand[12 * c + 4 * r + 3] = (c & 2) ? -t[r] : t[r];
        }
}

__global__ void __launch_bounds__(ES_POINT_THREADS)
essential_cheirality_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, const double* __restrict__ aux, const uint8_t* __restrict__ inl,
                            const EssResult* __restrict__ res, const double* __restrict__ cand, double dist, uint8_t* __restrict__ bits,
                            int32_t* __restrict__ cnt4) {
    const int i = blockIdx.x * ES_POINT_THREADS + threadIdx.x;
    unsigned bm = 0;
    if (i < n && res->found && inl[i]) {
        const double f = aux[0], cx = aux[1], cy = aux[2];
        const double x1 = ((double)a[2 * i] - cx) / f, y1 = ((double)a[2 * i + 1] - cy) / f;
        const double x2 = ((double)b[2 * i] - cx) / f, y2 = ((double)b[2 * i + 1] - cy) / f;
        for (int c = 0; c < 4; ++c) {
            const double* P = cand + 12 * c;
            // cv::triangulatePoints rows x P[2] - P[0], y P[2] - P[1] for P0 = [I|0] and P
            double A[4][4] = {{-1.0, 0.0, x1, 0.0}, {0.0, -1.0, y1, 0.0}, {0, 0, 0, 0}, {0, 0, 0, 0}}, Q[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) { A[2][k] = x2 * P[8 + k] - P[k]; A[3][k] = y2 * P[8 + k] - P[4 + k]; }
            if (!null_vector_fast(A, Q)) null_vector_4x4(A, Q);
            // recoverPose: Q2 Q3 > 0, Q /= Q3, depth < dist in the first camera, 0 < (P Q).z < dist in the second
            bool ok = Q[2] * Q[3] > 0.0;
            const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3];
            ok = ok && Z < dist;
            const double z2 = P[8] * X + P[9] * Y + P[10] * Z + P[11];
            ok = ok && z2 > 0.0 && z2 < dist;
            bm |= (ok ? 1u : 0u) << c;
        }
    }
    if (i < n) bits[i] = (uint8_t)bm;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const unsigned v = __ballot_sync(0xffffffffu, (bm >> c) & 1u);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(cnt4 + c, __popc(v));
    }
}

__global__ void __launch_bounds__(ES_POINT_THREADS)
essential_pose_kernel(const uint8_t* __restrict__ bits, int n, const int32_t* __restrict__ cnt4, const double* __restrict__ cand, EssResult* __restrict__ res,
                      uint8_t* __restrict__ pose_mask) {
    const int g0 = cnt4[0], g1 = cnt4[1], g2 = cnt4[2], g3 = cnt4[3];
    const int c = (g0 >= g1 && g0 >= g2 && g0 >= g3) ? 0 : (g1 >= g0 && g1 >= g2 && g1 >= g3) ? 1 : (g2 >= g0 && g2 >= g1 && g2 >= g3) ? 2 : 3;
    const int i = blockIdx.x * ES_POINT_THREADS + threadIdx.x;
    if (i < n) pose_mask[i] = (bits[i] >> c) & 1;
    if (i == 0 && res->found) {
        for (int r = 0; r < 3; ++r) {
            for (int q = 0; q < 3; ++q) res->R[3 * r + q] = cand[12 * c + 4 * r + q];
            res->t[r] = cand[12 * c + 4 * r + 3];
        }
        res->n_good = c == 0 ? g0 : c == 1 ? g1 : c == 2 ? g2 : g3;
    }
}

}  // namespace

extern "C" {

void sfmb200_essential_default_options(sfmb200_essential_options* opt) {
    if (!opt) return;
    opt->max_iters = 1000; opt->confidence = 0.999; opt->threshold_px = 1.0; opt->distance_thresh = 50.0; opt->seed = 0;
}

int sfmb200_find_camera_matrices(sfmb200_ctx* ctx, const float* K, const float* pts_left, int n_left, const float* pts_right, int n_right,
                                 const int32_t* match_q, const int32_t* match_t, int m, const sfmb200_essential_options* opt,
                                 double* E, double* R, double* t, uint8_t* inlier_mask, uint8_t* pose_mask, sfmb200_essential_summary* summary) {
    if (!ctx || !K || m < 0 || n_left < 0 || n_right < 0) return SFMB200_ERR_INVALID;
    sfmb200_essential_options o;
    sfmb200_essential_default_options(&o);
    if (opt) o = *opt;
    if (o.max_iters < 1 || !(o.confidence > 0.0 && o.confidence < 1.0) || !(o.threshold_px > 0.0) || !(o.distance_thresh > 0.0))
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "essential options: max_iters >= 1, confidence in (0, 1), threshold_px > 0, distance_thresh > 0");
    if ((size_t)o.max_iters * 10 > (size_t)INT32_MAX / 2) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "max_iters too large");
    const double focal = (double)K[0], cx = (double)K[2], cy = (double)K[5];
    if (!(focal != 0.0) || !std::isfinite(focal) || !std::isfinite(cx) || !std::isfinite(cy)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "K: focal length must be finite and nonzero");
    sfmb200_essential_summary sm;
    memset(&sm, 0, sizeof sm);
    if (summary) *summary = sm;
    if (E) memset(E, 0, 9 * sizeof(double));
    if (R) memset(R, 0, 9 * sizeof(double));
    if (t) memset(t, 0, 3 * sizeof(double));
    if (inlier_mask) memset(inlier_mask, 0, (size_t)m);
    if (pose_mask) memset(pose_mask, 0, (size_t)m);
    if (m > 0 && (!pts_left || !pts_right)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if ((match_q == nullptr) != (match_t == nullptr)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_q and match_t must both be given or both be NULL");
    if (!match_q && (m > n_left || m > n_right)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "identity alignment needs m <= min(n_left, n_right)");
    if (match_q)
        for (int i = 0; i < m; ++i)
            if (match_q[i] < 0 || match_q[i] >= n_left || match_t[i] < 0 || match_t[i] >= n_right)
                return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match %d indexes outside the keypoint arrays", i);
    if (m < 5) return SFMB200_OK;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const int S = m == 5 ? 1 : o.max_iters;       // five correspondences: every sample would hold the same five points
    const size_t slots = 10 * (size_t)S;
    // pinned staging: aux (f, cx, cy, 0...) | a | b on the way in; result | inlier mask | pose mask on the way out
    const size_t in_bytes = 80 + 16 * (size_t)m, out_bytes = Carver::pad(sizeof(EssResult)) + 2 * (size_t)m;
    SFM_CUDA(ctx, ctx->pinned.reserve(Carver::pad(in_bytes) + out_bytes));
    char* pin = (char*)ctx->pinned.p;
    double* aux = (double*)pin;
    for (int k = 0; k < 10; ++k) aux[k] = 0.0;
    aux[0] = focal; aux[1] = cx; aux[2] = cy;
    float* ha = (float*)(pin + 80);
    float* hb = ha + 2 * (size_t)m;
    for (int i = 0; i < m; ++i) {
        const int iq = match_q ? match_q[i] : i, it = match_t ? match_t[i] : i;
        ha[2 * i] = pts_left[2 * (size_t)iq]; ha[2 * i + 1] = pts_left[2 * (size_t)iq + 1];
        hb[2 * i] = pts_right[2 * (size_t)it]; hb[2 * i + 1] = pts_right[2 * (size_t)it + 1];
    }
    char* hout = pin + Carver::pad(in_bytes);
    EssResult* hres = (EssResult*)hout;
    uint8_t* hinl = (uint8_t*)(hout + Carver::pad(sizeof(EssResult)));
    uint8_t* hpose = hinl + m;

    const size_t bytes = Carver::pad(in_bytes) + Carver::pad(sizeof(Model) * slots) + Carver::pad(sizeof(EssResult)) + Carver::pad(4 * 12 * 8) +
                         Carver::pad(16) + 3 * Carver::pad((size_t)m) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    char* d_in = cv.take<char>(in_bytes);
    const double* d_aux = (const double*)d_in;
    const float* d_a = (const float*)(d_in + 80);
    const float* d_b = d_a + 2 * (size_t)m;
    Model* d_hyp = cv.take<Model>(slots);
    EssResult* d_res = cv.take<EssResult>(1);
    double* d_cand = cv.take<double>(48);
    int32_t* d_cnt4 = cv.take<int32_t>(4);
    uint8_t* d_inl = cv.take<uint8_t>(m);
    uint8_t* d_bits = cv.take<uint8_t>(m);
    uint8_t* d_pose = cv.take<uint8_t>(m);
    SFM_CUDA(ctx, ctx->ess_trace.reserve(Carver::pad(4 * 5 * (size_t)S) + Carver::pad(4 * (size_t)S) + Carver::pad(4 * slots) + 1024));
    Carver tc(ctx->ess_trace.p);
    int32_t* d_samples = tc.take<int32_t>(5 * (size_t)S);
    int32_t* d_nsol = tc.take<int32_t>(S);
    int32_t* d_counts = tc.take<int32_t>(slots);
    ctx->ess_trace_samples = 0;

    SFM_CUDA(ctx, cudaMemcpyAsync(d_in, pin, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    essential_solve_kernel<<<ceil_div(S, ES_SOLVE_THREADS), ES_SOLVE_THREADS, 0, ctx->stream>>>(d_a, d_b, m, S, o.seed, focal, cx, cy, d_samples, d_nsol, d_hyp);
    SFM_LAUNCH_CHECK(ctx);
    const float t2 = (float)((o.threshold_px / focal) * (o.threshold_px / focal));      // findEssentialMat: threshold /= focal
    essential_score_kernel<<<(unsigned)slots, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, m, d_hyp, d_nsol, d_aux, t2, d_counts);
    SFM_LAUNCH_CHECK(ctx);
    essential_select_kernel<<<1, 32, 0, ctx->stream>>>(d_nsol, d_counts, d_hyp, S, m, o.max_iters, o.confidence, d_res, d_cand, d_cnt4);
    SFM_LAUNCH_CHECK(ctx);
    const int pb = ceil_div(m, ES_POINT_THREADS);
    ransac_mask_kernel<1><<<ceil_div(m, RS_THREADS), RS_THREADS, 0, ctx->stream>>>(d_a, d_b, m, d_hyp, d_aux, t2, &d_res->best_slot, d_inl);
    SFM_LAUNCH_CHECK(ctx);
    essential_cheirality_kernel<<<pb, ES_POINT_THREADS, 0, ctx->stream>>>(d_a, d_b, m, d_aux, d_inl, d_res, d_cand, o.distance_thresh, d_bits, d_cnt4);
    SFM_LAUNCH_CHECK(ctx);
    essential_pose_kernel<<<pb, ES_POINT_THREADS, 0, ctx->stream>>>(d_bits, m, d_cnt4, d_cand, d_res, d_pose);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaMemcpyAsync(hres, d_res, sizeof(EssResult), cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(hinl, d_inl, (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(hpose, d_pose, (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->ess_trace_samples = S;

    sm.found = hres->found; sm.n_inliers = hres->n_inliers; sm.n_good = hres->n_good; sm.iterations = hres->iterations;
    sm.n_samples = S; sm.n_hypotheses = hres->n_hypotheses;
    if (summary) *summary = sm;
    if (!hres->found) return SFMB200_OK;
    if (E) memcpy(E, hres->E, 9 * sizeof(double));
    if (R) memcpy(R, hres->R, 9 * sizeof(double));
    if (t) memcpy(t, hres->t, 3 * sizeof(double));
    if (inlier_mask) memcpy(inlier_mask, hinl, (size_t)m);
    if (pose_mask) memcpy(pose_mask, hpose, (size_t)m);
    return SFMB200_OK;
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
