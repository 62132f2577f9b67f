// ransac.cu -- SURVEY.md 8 row f-2: batched hypothesis scoring for the three RANSAC stages that sit on either side of
// triangulation in the reference driver:
//   findHomographyInliers        SfMToyLib/SfMStereoUtilities.cpp:51-72   cv::findHomography(RANSAC, 10 px)   -> inlier count
//   findCameraMatricesFromMatch  SfMToyLib/SfMStereoUtilities.cpp:74-118  cv::findEssentialMat(RANSAC, 0.999, 1 px) + recoverPose
//   findCameraPoseFrom2D3DMatch  SfMToyLib/SfMStereoUtilities.cpp:208-243 cv::solvePnPRansac(100 iterations, 10 px, 0.99)
// OpenCV's RANSAC evaluates one hypothesis at a time over all correspondences (RANSACPointSetRegistrator::run -> computeError
// -> findInliers); here ALL hypotheses of a run are scored against ALL correspondences in one launch: grid (point chunks,
// hypotheses), a block counts the inliers of its chunk, integer atomics collect the counts (deterministic), a second kernel
// picks the best hypothesis (most inliers, ties -> lowest index = the first one OpenCV would have kept) and writes its mask.
// The hypotheses themselves come from the host (minimal solvers); the error formulas and their arithmetic types follow
// OpenCV's computeError callbacks so that a hypothesis gets the inlier set cv:: gives it:
//   homography  fundam.cpp  HomographyEstimatorCallback::computeError: FLOAT  ww = 1/(h6 x + h7 y + 1), dx, dy, err = dx^2 + dy^2
//   essential   five-point.cpp EMEstimatorCallback::computeError: DOUBLE Sampson error (x2^T E x1)^2 / (|Ex1|_xy^2 + |E^T x2|_xy^2), stored as float
//   pose        solvepnp.cpp PnPRansacCallback::computeError: projection (double), float difference, squared norm
// inlier  <=>  err <= (float)(threshold^2)   (RANSACPointSetRegistrator::findInliers).
#include "ransac_score.cuh"

extern "C" int sfmb200_ransac_score(sfmb200_ctx* ctx, int model, const float* a, const float* b, int n, const double* hyp, int nh, const double* aux9,
                                    double threshold, int32_t* inlier_counts, int32_t* best_index, uint8_t* best_mask) {
    if (!ctx || model < 0 || model > 2 || n < 0 || nh < 0) return SFMB200_ERR_INVALID;
    if (best_index) *best_index = -1;
    if (n == 0 || nh == 0) { if (inlier_counts) for (int h = 0; h < nh; ++h) inlier_counts[h] = 0; if (best_mask) memset(best_mask, 0, (size_t)n); return SFMB200_OK; }
    if (!a || !b || !hyp) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const int adim = model == 2 ? 3 : 2, hdim = model == 2 ? 12 : 9;
    std::vector<Model> hm(nh);
    for (int h = 0; h < nh; ++h) {
        memset(hm[h].m, 0, sizeof hm[h].m);
        for (int k = 0; k < hdim; ++k) hm[h].m[k] = hyp[(size_t)h * hdim + k];
        if (model == 0) {                                   // cv:: keeps homographies normalised to h22 = 1 (the error formula assumes it)
            const double s = hm[h].m[8];
            if (s != 0.0 && s != 1.0) for (int k = 0; k < 9; ++k) hm[h].m[k] /= s;
        }
    }
    double aux[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (aux9) memcpy(aux, aux9, sizeof aux);
    const size_t bytes = Carver::pad(4 * (size_t)n * adim) + Carver::pad(8 * (size_t)n) + Carver::pad(sizeof(Model) * nh) + Carver::pad(72) + Carver::pad(4 * (size_t)nh) + Carver::pad(n) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    float* d_a = cv.take<float>((size_t)n * adim); float* d_b = cv.take<float>((size_t)n * 2); Model* d_h = cv.take<Model>(nh); double* d_aux = cv.take<double>(9);
    int32_t* d_cnt = cv.take<int32_t>(nh); int32_t* d_best = cv.take<int32_t>(2); uint8_t* d_mask = cv.take<uint8_t>(n);
    SFM_CUDA(ctx, cudaMemcpyAsync(d_a, a, 4 * (size_t)n * adim, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_b, b, 8 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_h, hm.data(), sizeof(Model) * nh, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_aux, aux, 72, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 4 * (size_t)nh, ctx->stream));
    const float t2 = (float)(threshold * threshold);
    // enough blocks to fill the machine: hypotheses x point chunks
    const int chunks = std::max(1, std::min(ceil_div(n, RS_THREADS), ceil_div(4 * ctx->sm_count, nh)));
    const int per_block = ceil_div(n, chunks);
    dim3 grid(ceil_div(n, per_block), nh);
    if (model == 0) ransac_score_kernel<0><<<grid, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, n, d_h, d_aux, t2, per_block, d_cnt);
    else if (model == 1) ransac_score_kernel<1><<<grid, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, n, d_h, d_aux, t2, per_block, d_cnt);
    else ransac_score_kernel<2><<<grid, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, n, d_h, d_aux, t2, per_block, d_cnt);
    SFM_LAUNCH_CHECK(ctx);
    ransac_best_kernel<<<1, 1024, 0, ctx->stream>>>(d_cnt, nh, d_best);
    SFM_LAUNCH_CHECK(ctx);
    if (best_mask) {
        const int mb = ceil_div(n, RS_THREADS);
        if (model == 0) ransac_mask_kernel<0><<<mb, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, n, d_h, d_aux, t2, d_best, d_mask);
        else if (model == 1) ransac_mask_kernel<1><<<mb, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, n, d_h, d_aux, t2, d_best, d_mask);
        else ransac_mask_kernel<2><<<mb, RS_THREADS, 0, ctx->stream>>>(d_a, d_b, n, d_h, d_aux, t2, d_best, d_mask);
        SFM_LAUNCH_CHECK(ctx);
        SFM_CUDA(ctx, cudaMemcpyAsync(best_mask, d_mask, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    int32_t hb[2] = {-1, 0};
    if (inlier_counts) SFM_CUDA(ctx, cudaMemcpyAsync(inlier_counts, d_cnt, 4 * (size_t)nh, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(hb, d_best, 8, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (best_index) *best_index = hb[0];
    return SFMB200_OK;
}
