// pose.cu -- K9: camera pose from 2D-3D matches on the device, PnP RANSAC with a least-squares refit (SURVEY.md 8 row f-2).
//
// Replaces SfMStereoUtilities::findCameraPoseFrom2D3DMatch (reference SfMToyLib/SfMStereoUtilities.cpp:208-243):
//   cv::solvePnPRansac(points3D, points2D, K, dist, rvec, t, false, 100, RANSAC_THRESHOLD, 0.99, inliers)
// in one call, four launches:
//   1. pose_solve_kernel   one thread per sample: draw 5 distinct correspondences (em_sample, the counter-based sampler of the
//                          essential-matrix RANSAC), EPnP in fp64 (pose_math.cuh) -> at most one [R|t] per sample
//   2. pose_score_kernel   one CTA per sample: is_inlier<SFMB200_MODEL_POSE> (ransac_score.cuh, the arithmetic sfmb200_ransac_score
//                          pins against cv2) over all correspondences; a CTA owns its count, so counts are deterministic without atomics
//   3. pose_select_kernel  one warp: OpenCV's sequential loop (RANSACPointSetRegistrator::run, model_points = 5) over the counts in
//                          sample order, seq_select_chunk of ransac_select.cuh, shared with the essential-matrix RANSAC
//   4. pose_refit_kernel   one CTA: the winner's inlier mask, then damped Gauss-Newton (Levenberg-Marquardt) on (angle-axis, t)
//                          minimising the summed squared pixel reprojection error over those inliers, with the residual and
//                          Jacobian of ba_math.cuh; block reductions of J^T J / J^T r, a 6 x 6 Cholesky in one thread
// One upload, one download, one host synchronisation per call.  Samples and counts stay on the device (ctx->pose_trace) for
// sfmb200_pose_last_trace.
#include "ransac_score.cuh"
#include "ba_math.cuh"
#include "essential_math.cuh"
#include "pose_math.cuh"

namespace {

constexpr int PO_SOLVE_THREADS = 32;     // one sample per thread: 100 samples spread over 4 SMs
constexpr int PO_SCORE_THREADS = 128;    // one sample per CTA
constexpr int PO_REFIT_THREADS = 256;    // one CTA for the mask and the refit
constexpr int PO_RED = 28;               // J^T J upper triangle (21), J^T r (6), cost (1)

struct PoseResult {
    double rvec[3], R[9], t[3];
    int32_t found, n_inliers, iterations, n_hypotheses, refined, best;
};

// The solver of one sample, not inlined so that the RANSAC and the sfmb200_epnp test hook run the same machine code.
__device__ __noinline__ bool pose_solve_one(const double (*X)[3], const double (*uv)[2], const double* K, double* P) {
    double R[9], t[3];
    const bool ok = pm_epnp(X, uv, K[0], K[4], K[2], K[5], R, t);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) P[4 * r + c] = ok ? R[3 * r + c] : 0.0;
        P[4 * r + 3] = ok ? t[r] : 0.0;
    }
    return ok;
}

__global__ void __launch_bounds__(PO_SOLVE_THREADS)
pose_solve_kernel(const float* __restrict__ X, const float* __restrict__ uv, int m, int S, uint64_t seed, const double* __restrict__ K,
                  int32_t* __restrict__ samples, int32_t* __restrict__ nsol, Model* __restrict__ hyp) {
    const int s = blockIdx.x * PO_SOLVE_THREADS + threadIdx.x;
    if (s >= S) return;
    int idx[PM_N];
    em_sample(seed, (uint32_t)s, m, idx);
    double Xs[PM_N][3], us[PM_N][2], k[9];
    for (int q = 0; q < 9; ++q) k[q] = K[q];
    for (int j = 0; j < PM_N; ++j) {
        for (int c = 0; c < 3; ++c) Xs[j][c] = (double)X[3 * (size_t)idx[j] + c];
        us[j][0] = (double)uv[2 * (size_t)idx[j]]; us[j][1] = (double)uv[2 * (size_t)idx[j] + 1];
        samples[PM_N * s + j] = idx[j];
    }
    double P[12];
    nsol[s] = pose_solve_one(Xs, us, k, P) ? 1 : 0;
    for (int q = 0; q < 12; ++q) hyp[s].m[q] = P[q];
}

__global__ void __launch_bounds__(PO_SOLVE_THREADS)
epnp_kernel(const double* __restrict__ X, const double* __restrict__ uv, const double* __restrict__ K, int ns, double* __restrict__ Rt,
            uint8_t* __restrict__ ok) {
    const int s = blockIdx.x * PO_SOLVE_THREADS + threadIdx.x;
    if (s >= ns) return;
    double Xs[PM_N][3], us[PM_N][2], k[9], P[12];
    for (int q = 0; q < 9; ++q) k[q] = K[q];
    for (int j = 0; j < PM_N; ++j) {
        for (int c = 0; c < 3; ++c) Xs[j][c] = X[15 * (size_t)s + 3 * j + c];
        us[j][0] = uv[10 * (size_t)s + 2 * j]; us[j][1] = uv[10 * (size_t)s + 2 * j + 1];
    }
    ok[s] = pose_solve_one(Xs, us, k, P) ? 1 : 0;
    for (int q = 0; q < 12; ++q) Rt[12 * (size_t)s + q] = P[q];
}

__global__ void __launch_bounds__(PO_SCORE_THREADS)
pose_score_kernel(const float* __restrict__ X, const float* __restrict__ uv, int m, const Model* __restrict__ hyp, const int32_t* __restrict__ nsol,
                  const double* __restrict__ K, float t2, int32_t* __restrict__ counts) {
    constexpr int W = PO_SCORE_THREADS / 32;
    __shared__ double M[12], A[9];
    __shared__ int wsum[W];
    const int s = blockIdx.x;
    if (threadIdx.x < 12) M[threadIdx.x] = hyp[s].m[threadIdx.x];
    if (threadIdx.x < 9) A[threadIdx.x] = K[threadIdx.x];
    __syncthreads();
    const bool has = nsol[s] != 0;
    int c = 0;
    for (int i = threadIdx.x; has && i < m; i += PO_SCORE_THREADS) c += is_inlier<SFMB200_MODEL_POSE>(M, A, X, uv, i, t2) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int v = 0;
        for (int w = 0; w < W; ++w) v += wsum[w];
        counts[s] = has ? v : -1;                       // -1: the sample gave no pose
    }
}

__global__ void __launch_bounds__(32)
pose_select_kernel(const int32_t* __restrict__ nsol, const int32_t* __restrict__ counts, int S, int m, int max_iters, double confidence,
                   PoseResult* __restrict__ res) {
    __shared__ int32_t sn[32], sc[32];
    const int lane = threadIdx.x;
    SeqSelect st;
    seq_select_begin(st, max_iters);
    int nh = 0;
    for (int base = 0; base < S; base += 32) {
        const int k = min(32, S - base);
        const int v = lane < k ? nsol[base + lane] : 0;
        nh += v;
        if (!__shfl_sync(0xffffffffu, st.iter < st.niters, 0)) continue;    // the loop has stopped: only the hypothesis total is left
        sn[lane] = v;
        sc[lane] = lane < k ? counts[base + lane] : 0;
        __syncwarp();
        if (lane == 0) seq_select_chunk(st, sn, sc, 1, k, m, confidence, PM_N, 0);
        __syncwarp();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nh += __shfl_xor_sync(0xffffffffu, nh, o);
    if (lane != 0) return;
    if (m == PM_N) {             // solvePnPRansac's model_points == npoints branch: EPnP on the five points, every point an inlier
        st.best = nsol[0] ? 0 : -1; st.max_good = nsol[0] ? PM_N : 0; st.iter = 1;
    }
    res->found = st.best >= 0 ? 1 : 0;
    res->best = st.best;
    res->n_inliers = st.best >= 0 ? st.max_good : 0;
    res->iterations = st.iter;
    res->n_hypotheses = nh;
    res->refined = 0;
}

// Sums over the inliers at the parameters x (angle-axis, t) of the rows r = (fx (x/z - xn), fy (y/z - yn)): J^T J upper
// triangle, J^T r and the cost (jac = true), or the cost only; the CTA total lands in out[0 .. PO_RED) (cost in out[27]),
// summed in a fixed order.
__device__ void pose_accumulate(const float* __restrict__ X, const float* __restrict__ uv, int m, const uint8_t* __restrict__ mask,
                                const double* K, const double* x, bool jac, double (*red)[PO_RED], double* out) {
    CamDerived d;
    cam_derive(x, d);
    const double fx = K[0], fy = K[4], cx = K[2], cy = K[5];
    double acc[PO_RED];
#pragma unroll
    for (int k = 0; k < PO_RED; ++k) acc[k] = 0.0;
    for (int i = threadIdx.x; i < m; i += PO_REFIT_THREADS) {
        if (!mask[i]) continue;
        const double Xd[3] = {(double)X[3 * (size_t)i], (double)X[3 * (size_t)i + 1], (double)X[3 * (size_t)i + 2]};
        const double xn = ((double)uv[2 * (size_t)i] - cx) / fx, yn = ((double)uv[2 * (size_t)i + 1] - cy) / fy;
        double r[2];
        if (jac) {
            double Jc[12], Jp[6], Jf[2];
            obs_eval(d, Xd, 1.0, xn, yn, r, Jc, Jp, Jf);
            double J0[6], J1[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) { J0[k] = fx * Jc[k]; J1[k] = fy * Jc[6 + k]; }
            r[0] *= fx; r[1] *= fy;
            int o = 0;
#pragma unroll
            for (int a = 0; a < 6; ++a) {
#pragma unroll
                for (int b = a; b < 6; ++b) acc[o++] += J0[a] * J0[b] + J1[a] * J1[b];
            }
#pragma unroll
            for (int a = 0; a < 6; ++a) acc[21 + a] += J0[a] * r[0] + J1[a] * r[1];
        } else {
            obs_residual(d, Xd, 1.0, xn, yn, r);
            r[0] *= fx; r[1] *= fy;
        }
        acc[27] += r[0] * r[0] + r[1] * r[1];
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < PO_RED; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[w][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < PO_RED) {
        double v = 0.0;
        for (int q = 0; q < PO_REFIT_THREADS / 32; ++q) v += red[q][threadIdx.x];
        out[threadIdx.x] = v;
    }
    __syncthreads();
}

// (A + lambda diag(A)) dx = -g with A the packed upper triangle of J^T J: Cholesky, false when not positive definite
__device__ bool pose_damped_solve(const double* Ap, const double* g, double lambda, double* dx) {
    double A[6][6], L[6][6];
    int o = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) { A[a][b] = A[b][a] = Ap[o++]; }
    for (int a = 0; a < 6; ++a) A[a][a] += lambda * A[a][a];
    for (int j = 0; j < 6; ++j) {
        double s = A[j][j];
        for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
        if (!(s > 0.0)) return false;
        L[j][j] = sqrt(s);
        for (int i = j + 1; i < 6; ++i) {
            double v = A[i][j];
            for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
            L[i][j] = v / L[j][j];
        }
    }
    double y[6];
    for (int i = 0; i < 6; ++i) {
        double v = -g[i];
        for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
        y[i] = v / L[i][i];
    }
    for (int i = 5; i >= 0; --i) {
        double v = y[i];
        for (int k = i + 1; k < 6; ++k) v -= L[k][i] * dx[k];
        dx[i] = v / L[i][i];
    }
    for (int i = 0; i < 6; ++i)
        if (!pm_finite(dx[i])) return false;
    return true;
}

__global__ void __launch_bounds__(PO_REFIT_THREADS)
pose_refit_kernel(const float* __restrict__ X, const float* __restrict__ uv, int m, const Model* __restrict__ hyp, const double* __restrict__ Kg,
                  float t2, int refine_iters, PoseResult* __restrict__ res, uint8_t* __restrict__ mask) {
    __shared__ double P[12], K[9], x[6], xc[6], sA[PO_RED], sB[PO_RED];
    __shared__ double red[PO_REFIT_THREADS / 32][PO_RED];
    __shared__ int s_stop, s_refit;
    const int found = res->found, best = res->best;
    if (!found) {
        for (int i = threadIdx.x; i < m; i += PO_REFIT_THREADS) mask[i] = 0;
        return;
    }
    if (threadIdx.x < 12) P[threadIdx.x] = hyp[best].m[threadIdx.x];
    if (threadIdx.x < 9) K[threadIdx.x] = Kg[threadIdx.x];
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += PO_REFIT_THREADS)
        mask[i] = (m == PM_N || is_inlier<SFMB200_MODEL_POSE>(P, K, X, uv, i, t2)) ? 1 : 0;
    if (threadIdx.x == 0) {
        const double R[9] = {P[0], P[1], P[2], P[4], P[5], P[6], P[8], P[9], P[10]};
        pm_rotmat_to_aa(R, x);
        x[3] = P[3]; x[4] = P[7]; x[5] = P[11];
        s_refit = m > PM_N && res->n_inliers >= 6 && refine_iters > 0;
        s_stop = 0;
    }
    __syncthreads();                         // the mask and x are visible to the whole CTA
    bool refined = false;
    if (s_refit) {
        double lambda = 1e-3, cost0 = 0.0, cost = 0.0;       // thread 0's copies
        bool need_jac = true;
        for (int it = 0; it < refine_iters; ++it) {
            if (need_jac) pose_accumulate(X, uv, m, mask, K, x, true, red, sA);
            if (threadIdx.x == 0) {
                if (it == 0) cost0 = cost = sA[27];
                double dx[6];
                const bool ok = pose_damped_solve(sA, sA + 21, lambda, dx);
                for (int k = 0; k < 6; ++k) xc[k] = ok ? x[k] + dx[k] : x[k];
                s_stop = ok ? 0 : 2;
            }
            __syncthreads();
            pose_accumulate(X, uv, m, mask, K, xc, false, red, sB);
            if (threadIdx.x == 0) {
                double dn = 0.0, xn = 0.0;
                for (int k = 0; k < 6; ++k) { dn += (xc[k] - x[k]) * (xc[k] - x[k]); xn += x[k] * x[k]; }
                const bool small_step = sqrt(dn) <= 1e-10 * (sqrt(xn) + 1e-10);
                if (s_stop == 0 && sB[27] < cost) {
                    const bool small_drop = cost - sB[27] <= 1e-10 * cost;
                    for (int k = 0; k < 6; ++k) x[k] = xc[k];
                    cost = sB[27]; refined = true; need_jac = true;
                    lambda = fmax(lambda * 0.1, 1e-12);
                    s_stop = small_step || small_drop;
                } else {
                    lambda *= 10.0; need_jac = false;
                    s_stop = small_step || lambda > 1e12;
                }
            }
            __syncthreads();
            need_jac = __syncthreads_or(threadIdx.x == 0 && need_jac);
            if (s_stop) break;
        }
        refined = threadIdx.x == 0 && refined && cost < cost0;
    }
    if (threadIdx.x != 0) return;
    PoseResult& r = *res;
    r.refined = refined ? 1 : 0;
    if (refined) {
        CamDerived d;
        cam_derive(x, d);
        for (int k = 0; k < 9; ++k) r.R[k] = d.R[k];
        for (int k = 0; k < 3; ++k) { r.rvec[k] = x[k]; r.t[k] = x[3 + k]; }
    } else {                                 // the RANSAC pose
        const double R[9] = {P[0], P[1], P[2], P[4], P[5], P[6], P[8], P[9], P[10]};
        for (int k = 0; k < 9; ++k) r.R[k] = R[k];
        pm_rotmat_to_aa(R, r.rvec);
        r.t[0] = P[3]; r.t[1] = P[7]; r.t[2] = P[11];
    }
}

int po_check(sfmb200_ctx* ctx, const sfmb200_pose_options& o, const float* K) {
    if (o.max_iters < 1 || o.max_iters > (1 << 24) || !(o.confidence > 0.0 && o.confidence < 1.0) || !(o.threshold_px > 0.0) ||
        !std::isfinite(o.threshold_px) || o.refine_iters < 0)
        return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "pose options: max_iters in [1, 2^24], confidence in (0, 1), finite threshold_px > 0, refine_iters >= 0");
    if (!K) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    for (int q = 0; q < 9; ++q)
        if (!std::isfinite(K[q])) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "K: entries must be finite");
    if (!(K[0] > 0.0f) || !(K[4] > 0.0f)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "K: fx and fy must be > 0");
    return SFMB200_OK;
}

}  // namespace

extern "C" {

void sfmb200_pose_default_options(sfmb200_pose_options* opt) {
    if (!opt) return;
    opt->max_iters = 100; opt->confidence = 0.99; opt->threshold_px = 10.0; opt->refine_iters = 20; opt->seed = 0;
}

int sfmb200_find_camera_pose(sfmb200_ctx* ctx, const float* K, const float* pts3, const float* pts2, int m, const sfmb200_pose_options* opt,
                             double* rvec, double* R, double* t, uint8_t* inlier_mask, sfmb200_pose_summary* summary) {
    if (!ctx) return SFMB200_ERR_INVALID;
    sfmb200_pose_options o;
    sfmb200_pose_default_options(&o);
    if (opt) o = *opt;
    if (const int rc = po_check(ctx, o, K)) return rc;
    if (m < 0) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "m must be >= 0");
    if (m > 0 && (!pts3 || !pts2)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (summary) memset(summary, 0, sizeof(sfmb200_pose_summary));
    if (rvec) memset(rvec, 0, 3 * sizeof(double));
    if (R) memset(R, 0, 9 * sizeof(double));
    if (t) memset(t, 0, 3 * sizeof(double));
    if (inlier_mask) memset(inlier_mask, 0, (size_t)m);
    if (m < PM_N) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->pose_trace_samples = 0;
        return SFMB200_OK;
    }
    const int S = m == PM_N ? 1 : o.max_iters;           // five correspondences: every sample would hold the same five points

    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    // pinned staging: K | X | uv on the way in; result | mask on the way out.  The device carving has the same layout.
    const size_t in_bytes = Carver::pad(72) + Carver::pad(12 * (size_t)m) + Carver::pad(8 * (size_t)m);
    const size_t out_bytes = Carver::pad(sizeof(PoseResult)) + Carver::pad((size_t)m);
    SFM_CUDA(ctx, ctx->pinned.reserve(in_bytes + out_bytes + 256));
    Carver hc(ctx->pinned.p);
    double* h_K = hc.take<double>(9);
    float* h_X = hc.take<float>(3 * (size_t)m);
    float* h_uv = hc.take<float>(2 * (size_t)m);
    PoseResult* h_res = hc.take<PoseResult>(1);
    uint8_t* h_mask = hc.take<uint8_t>((size_t)m);
    const size_t in_len = (char*)h_uv + 8 * (size_t)m - (char*)ctx->pinned.p;
    const size_t out_off = (char*)h_res - (char*)ctx->pinned.p, out_len = hc.off - out_off;
    for (int q = 0; q < 9; ++q) h_K[q] = (double)K[q];
    memcpy(h_X, pts3, 12 * (size_t)m);
    memcpy(h_uv, pts2, 8 * (size_t)m);

    SFM_CUDA(ctx, ctx->scratch.reserve(in_bytes + out_bytes + Carver::pad(4 * (size_t)S) + Carver::pad(sizeof(Model) * S) + 1024));
    Carver cv(ctx->scratch.p);
    const double* d_K = cv.take<double>(9);
    const float* d_X = cv.take<float>(3 * (size_t)m);
    const float* d_uv = cv.take<float>(2 * (size_t)m);
    PoseResult* d_res = cv.take<PoseResult>(1);
    uint8_t* d_mask = cv.take<uint8_t>((size_t)m);
    int32_t* d_nsol = cv.take<int32_t>(S);
    Model* d_hyp = cv.take<Model>(S);
    SFM_CUDA(ctx, ctx->pose_trace.reserve(Carver::pad(4 * PM_N * (size_t)S) + Carver::pad(4 * (size_t)S) + 512));
    Carver tc(ctx->pose_trace.p);
    int32_t* d_samples = tc.take<int32_t>(PM_N * (size_t)S);
    int32_t* d_counts = tc.take<int32_t>(S);
    ctx->pose_trace_samples = 0;

    SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, ctx->pinned.p, in_len, cudaMemcpyHostToDevice, ctx->stream));
    const float t2 = (float)(o.threshold_px * o.threshold_px);
    pose_solve_kernel<<<ceil_div(S, PO_SOLVE_THREADS), PO_SOLVE_THREADS, 0, ctx->stream>>>(d_X, d_uv, m, S, o.seed, d_K, d_samples, d_nsol, d_hyp);
    SFM_LAUNCH_CHECK(ctx);
    pose_score_kernel<<<S, PO_SCORE_THREADS, 0, ctx->stream>>>(d_X, d_uv, m, d_hyp, d_nsol, d_K, t2, d_counts);
    SFM_LAUNCH_CHECK(ctx);
    pose_select_kernel<<<1, 32, 0, ctx->stream>>>(d_nsol, d_counts, S, m, o.max_iters, o.confidence, d_res);
    SFM_LAUNCH_CHECK(ctx);
    pose_refit_kernel<<<1, PO_REFIT_THREADS, 0, ctx->stream>>>(d_X, d_uv, m, d_hyp, d_K, t2, o.refine_iters, d_res, d_mask);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaMemcpyAsync((char*)ctx->pinned.p + out_off, (char*)ctx->scratch.p + out_off, out_len, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->pose_trace_samples = S;

    const PoseResult& r = *h_res;
    if (summary) {
        summary->found = r.found; summary->n_inliers = r.n_inliers; summary->iterations = r.iterations; summary->n_samples = S;
        summary->n_hypotheses = r.n_hypotheses; summary->refined = r.refined;
    }
    if (!r.found) return SFMB200_OK;
    if (rvec) memcpy(rvec, r.rvec, 3 * sizeof(double));
    if (R) memcpy(R, r.R, 9 * sizeof(double));
    if (t) memcpy(t, r.t, 3 * sizeof(double));
    if (inlier_mask) memcpy(inlier_mask, h_mask, (size_t)m);
    return SFMB200_OK;
}

int sfmb200_epnp(sfmb200_ctx* ctx, const double* X, const double* uv, const double* K, int ns, double* Rt, uint8_t* ok) {
    if (!ctx || ns < 0) return SFMB200_ERR_INVALID;
    if (ns == 0) return SFMB200_OK;
    if (!X || !uv || !K || !Rt || !ok) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t bytes = Carver::pad(120 * (size_t)ns) + Carver::pad(80 * (size_t)ns) + Carver::pad(72) + Carver::pad(96 * (size_t)ns) +
                         Carver::pad((size_t)ns) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    double* d_X = cv.take<double>(15 * (size_t)ns); double* d_uv = cv.take<double>(10 * (size_t)ns); double* d_K = cv.take<double>(9);
    double* d_Rt = cv.take<double>(12 * (size_t)ns); uint8_t* d_ok = cv.take<uint8_t>((size_t)ns);
    SFM_CUDA(ctx, cudaMemcpyAsync(d_X, X, 120 * (size_t)ns, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_uv, uv, 80 * (size_t)ns, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_K, K, 72, cudaMemcpyHostToDevice, ctx->stream));
    epnp_kernel<<<ceil_div(ns, PO_SOLVE_THREADS), PO_SOLVE_THREADS, 0, ctx->stream>>>(d_X, d_uv, d_K, ns, d_Rt, d_ok);
    SFM_LAUNCH_CHECK(ctx);
    SFM_CUDA(ctx, cudaMemcpyAsync(Rt, d_Rt, 96 * (size_t)ns, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(ok, d_ok, (size_t)ns, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SFMB200_OK;
}

int sfmb200_pose_last_trace(sfmb200_ctx* ctx, int cap, int32_t* samples, int32_t* counts) {
    if (!ctx || cap < 0) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    const int S = ctx->pose_trace_samples;
    const int k = cap < S ? cap : S;
    if (k == 0) return S;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
    Carver tc(ctx->pose_trace.p);
    int32_t* d_samples = tc.take<int32_t>(PM_N * (size_t)S);
    int32_t* d_counts = tc.take<int32_t>(S);
    if (samples && cudaMemcpyAsync(samples, d_samples, 4 * PM_N * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (counts && cudaMemcpyAsync(counts, d_counts, 4 * (size_t)k, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return -1;
    return S;
}

}  // extern "C"
