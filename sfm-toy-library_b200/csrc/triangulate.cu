// triangulate.cu -- K2: batched two-view DLT triangulation with fused gather / normalise / reproject / filter.
//
// Replaces SfMStereoUtilities::triangulateViews (reference SfMToyLib/SfMStereoUtilities.cpp:120-206) and the gather of
// GetAlignedPointsFromMatch (reference SfMToyLib/SfMCommon.cpp:63-87), which the reference executes as six OpenCV calls:
//   undistortPoints x2 (:146-147) -> triangulatePoints (:150) -> convertPointsFromHomogeneous (:153)
//   -> Rodrigues + projectPoints x2 (:155-167) -> 10 px reprojection filter in either view (:184-203).
// One thread per match does all of it in registers: indexed load of the two keypoints (the descriptor-row copies of
// SfMCommon.cpp:78,80 are dead work and are dropped), x_n = (u - c) * (1/f) in double rounded to float (what
// cv::undistortPoints returns), the 4x4 DLT matrix in double, its smallest right singular vector by one-sided
// (Hestenes) Jacobi in double -- the algorithm cv::SVD uses -- float dehomogenisation with a float reciprocal,
// double projection with the float-rvec round-tripped rotation, float pixel error, keep flag.
// HBM traffic: 16 B in (+8 B indices) and 13 B out per match; everything else lives in registers.
// sfmb200_triangulate_pairs runs the same kernel for many pairs: one upload of all key points and matches, one launch per pair
// with that pair's parameters and slices, one download.  It does not use a kernel of its own: ptxas decides per kernel which
// multiplies and adds it contracts into FMAs, so a second kernel with the same source rounds differently on some matches.
#include "common.cuh"
#include "dlt_math.cuh"
#include <cfloat>
#include <cmath>

namespace {

struct TriParams {
    double PL[12], PR[12];     // float poses widened (DLT rows)
    double RtL[12], RtR[12];   // [R|t] as cv::projectPoints sees them (float rvec round trip)
    double fx, fy, cx, cy, ifx, ify;
    float max_reproj;
};

__global__ void __launch_bounds__(128)
triangulate_kernel(TriParams P, const float2* __restrict__ ptsL, const float2* __restrict__ ptsR,
                   const int32_t* __restrict__ mq, const int32_t* __restrict__ mt, int m,
                   float* __restrict__ X, uint8_t* __restrict__ keep, int32_t* __restrict__ n_keep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int k = 0;
    if (i < m) {
        const int iq = mq ? mq[i] : i, it = mt ? mt[i] : i;
        const float2 l = __ldg(ptsL + iq), r = __ldg(ptsR + it);
        // cv::undistortPoints without distortion: (u - c) * (1/f) in double, returned as float
        const double xl = (double)(float)(((double)l.x - P.cx) * P.ifx), yl = (double)(float)(((double)l.y - P.cy) * P.ify);
        const double xr = (double)(float)(((double)r.x - P.cx) * P.ifx), yr = (double)(float)(((double)r.y - P.cy) * P.ify);
        double A[4][4], Xh[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            A[0][c] = xl * P.PL[8 + c] - P.PL[c];
            A[1][c] = yl * P.PL[8 + c] - P.PL[4 + c];
            A[2][c] = xr * P.PR[8 + c] - P.PR[c];
            A[3][c] = yr * P.PR[8 + c] - P.PR[4 + c];
        }
        if (!null_vector_fast(A, Xh)) null_vector_4x4(A, Xh);       // Jacobi SVD when the closed-form path declines
        // triangulatePoints returns float; convertPointsFromHomogeneous: scale = 1/w in float (w == 0 -> 1)
        const float hx = (float)Xh[0], hy = (float)Xh[1], hz = (float)Xh[2], hw = (float)Xh[3];
        const float sc = hw != 0.f ? __frcp_rn(hw) : 1.f;
        const float px = hx * sc, py = hy * sc, pz = hz * sc;
        X[3 * (size_t)i] = px; X[3 * (size_t)i + 1] = py; X[3 * (size_t)i + 2] = pz;
        // projectPoints in double, float pixel out; error norm in double of float differences
        double e2[2];
#pragma unroll
        for (int v = 0; v < 2; ++v) {
            const double* Rt = v == 0 ? P.RtL : P.RtR;
            const double Xc = Rt[0] * px + Rt[1] * py + Rt[2] * pz + Rt[3];
            const double Yc = Rt[4] * px + Rt[5] * py + Rt[6] * pz + Rt[7];
            double Zc = Rt[8] * px + Rt[9] * py + Rt[10] * pz + Rt[11];
            Zc = Zc != 0.0 ? 1.0 / Zc : 1.0;
            const float pu = (float)(Xc * Zc * P.fx + P.cx), pv = (float)(Yc * Zc * P.fy + P.cy);
            const float du = pu - (v == 0 ? l.x : r.x), dv = pv - (v == 0 ? l.y : r.y);
            e2[v] = sqrt((double)du * du + (double)dv * dv);
        }
        k = !(e2[0] > (double)P.max_reproj || e2[1] > (double)P.max_reproj);     // :186-187 (NaN compares false -> kept)
        keep[i] = (uint8_t)k;
    }
    // survivors: warp ballot -> one atomic per warp
    const unsigned b = __ballot_sync(0xffffffffu, k);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_keep, __popc(b));
}

// --- host: cv::Rodrigues(R) -> float rvec -> rotation matrix, i.e. the [R|t] projectPoints really uses (:155-167) ---
void rotmat_to_rvec(const double R[9], double r[3]) {
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = std::sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1.0) * 0.5;
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    const double theta = std::acos(c);
    if (s < 1e-5) {
        if (c > 0) { r[0] = r[1] = r[2] = 0; return; }
        double t;
        t = (R[0] + 1) * 0.5; rx = std::sqrt(t > 0 ? t : 0);
        t = (R[4] + 1) * 0.5; ry = std::sqrt(t > 0 ? t : 0) * (R[1] < 0 ? -1.0 : 1.0);
        t = (R[8] + 1) * 0.5; rz = std::sqrt(t > 0 ? t : 0) * (R[2] < 0 ? -1.0 : 1.0);
        if (std::fabs(rx) < std::fabs(ry) && std::fabs(rx) < std::fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
        const double n = theta / std::sqrt(rx * rx + ry * ry + rz * rz);
        r[0] = rx * n; r[1] = ry * n; r[2] = rz * n;
        return;
    }
    const double vth = theta / (2.0 * s);
    r[0] = rx * vth; r[1] = ry * vth; r[2] = rz * vth;
}

void pose_roundtrip(const float P[12], double Rt[12]) {
    double R[9], r[3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[3 * i + j] = (double)P[4 * i + j];
    rotmat_to_rvec(R, r);
    for (int i = 0; i < 3; ++i) r[i] = (double)(float)r[i];          // the rvec Mat is CV_32F
    const double theta = std::sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    double R2[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (theta >= DBL_EPSILON) {
        const double c = std::cos(theta), s = std::sin(theta), c1 = 1.0 - c, x = r[0] / theta, y = r[1] / theta, z = r[2] / theta;
        R2[0] = c + c1 * x * x;     R2[1] = c1 * x * y - s * z; R2[2] = c1 * x * z + s * y;
        R2[3] = c1 * x * y + s * z; R2[4] = c + c1 * y * y;     R2[5] = c1 * y * z - s * x;
        R2[6] = c1 * x * z - s * y; R2[7] = c1 * y * z + s * x; R2[8] = c + c1 * z * z;
    }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rt[4 * i + j] = R2[3 * i + j];
        Rt[4 * i + 3] = (double)P[4 * i + 3];
    }
}

void make_params(const float* K, const float* Pl, const float* Pr, float max_reproj, TriParams& P) {
    for (int i = 0; i < 12; ++i) { P.PL[i] = (double)Pl[i]; P.PR[i] = (double)Pr[i]; }
    pose_roundtrip(Pl, P.RtL); pose_roundtrip(Pr, P.RtR);
    P.fx = K[0]; P.fy = K[4]; P.cx = K[2]; P.cy = K[5];
    P.ifx = 1.0 / P.fx; P.ify = 1.0 / P.fy;
    P.max_reproj = max_reproj;
}

}  // namespace

static int triangulate_launch(sfmb200_ctx* ctx, const TriParams& P, const float* d_l, const float* d_r, const int32_t* d_mq,
                              const int32_t* d_mt, int m, float* d_X, uint8_t* d_keep, int32_t* d_n) {
    SFM_CUDA(ctx, cudaMemsetAsync(d_n, 0, sizeof(int32_t), ctx->stream));
    if (m == 0) return SFMB200_OK;
    triangulate_kernel<<<ceil_div(m, 128), 128, 0, ctx->stream>>>(P, (const float2*)d_l, (const float2*)d_r, d_mq, d_mt, m, d_X, d_keep, d_n);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

extern "C" {

int sfmb200_triangulate_device(sfmb200_ctx* ctx, const float* K, const float* Pl, const float* Pr, const float* d_l, const float* d_r,
                               const int32_t* d_mq, const int32_t* d_mt, int m, float max_reproj, float* d_X, uint8_t* d_keep, int32_t* d_n) {
    if (!ctx || !K || !Pl || !Pr || m < 0 || !d_n) return SFMB200_ERR_INVALID;
    if ((d_mq == nullptr) != (d_mt == nullptr)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "match_q and match_t must both be given or both be NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    TriParams P; make_params(K, Pl, Pr, max_reproj, P);
    return triangulate_launch(ctx, P, d_l, d_r, d_mq, d_mt, m, d_X, d_keep, d_n);
}

int sfmb200_triangulate(sfmb200_ctx* ctx, const float* K, const float* Pl, const float* Pr, const float* pts_left, int n_left,
                        const float* pts_right, int n_right, const int32_t* match_q, const int32_t* match_t, int m, float max_reproj,
                        float* X, uint8_t* keep, int* n_keep) {
    if (!ctx || !K || !Pl || !Pr || m < 0 || n_left < 0 || n_right < 0) return SFMB200_ERR_INVALID;
    if (n_keep) *n_keep = 0;
    if (m == 0) return SFMB200_OK;
    if (!pts_left || !pts_right || !X || !keep) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (const int rc = check_two_view_matches(ctx, match_q, match_t, m, n_left, n_right)) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t bytes = Carver::pad(8 * (size_t)n_left) + Carver::pad(8 * (size_t)n_right) + 2 * Carver::pad(4 * (size_t)m) +
                         Carver::pad(12 * (size_t)m) + Carver::pad(m) + 1024;
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver cv(ctx->scratch.p);
    float* d_l = cv.take<float>(2 * (size_t)n_left); float* d_r = cv.take<float>(2 * (size_t)n_right);
    int32_t* d_mq = cv.take<int32_t>(m); int32_t* d_mt = cv.take<int32_t>(m);
    float* d_X = cv.take<float>(3 * (size_t)m); uint8_t* d_keep = cv.take<uint8_t>(m); int32_t* d_n = cv.take<int32_t>(1);
    SFM_CUDA(ctx, cudaMemcpyAsync(d_l, pts_left, 8 * (size_t)n_left, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(d_r, pts_right, 8 * (size_t)n_right, cudaMemcpyHostToDevice, ctx->stream));
    if (match_q) {
        SFM_CUDA(ctx, cudaMemcpyAsync(d_mq, match_q, 4 * (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
        SFM_CUDA(ctx, cudaMemcpyAsync(d_mt, match_t, 4 * (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
    }
    TriParams P; make_params(K, Pl, Pr, max_reproj, P);
    int rc = triangulate_launch(ctx, P, d_l, d_r, match_q ? d_mq : nullptr, match_q ? d_mt : nullptr, m, d_X, d_keep, d_n);
    if (rc) return rc;
    int32_t hn = 0;
    SFM_CUDA(ctx, cudaMemcpyAsync(X, d_X, 12 * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(keep, d_keep, (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(&hn, d_n, 4, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (n_keep) *n_keep = hn;
    return SFMB200_OK;
}

int sfmb200_triangulate_pairs(sfmb200_ctx* ctx, const float* K, const float* poses, const float* pts, const int32_t* img_off, int n_img,
                              const int32_t* pairs, int n_pairs, const int32_t* match_q, const int32_t* match_t, const int64_t* match_off,
                              float max_reproj_px, float* X, uint8_t* keep, int32_t* n_keep) {
    if (!ctx || n_img < 0 || n_pairs < 0) return SFMB200_ERR_INVALID;
    if (n_pairs == 0) return SFMB200_OK;
    if (!K || !poses) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    int64_t M = 0;
    if (const int rc = check_pair_batch(ctx, pts, img_off, n_img, pairs, n_pairs, match_q, match_t, match_off, INT32_MAX, &M)) return rc;
    if (M > 0 && (!X || !keep)) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    if (n_keep) memset(n_keep, 0, sizeof(int32_t) * (size_t)n_pairs);
    if (M == 0) return SFMB200_OK;
    const int64_t NP = img_off[n_img];

    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    // pinned staging and device scratch share one layout: key points | match_q | match_t | n_keep | X | keep.  The upload runs up to
    // n_keep (zeroed here), the download from n_keep on.
    const size_t bytes = Carver::pad(8 * (size_t)NP) + 2 * Carver::pad(4 * (size_t)M) + Carver::pad(4 * (size_t)n_pairs) +
                         Carver::pad(12 * (size_t)M) + Carver::pad((size_t)M) + 256;
    SFM_CUDA(ctx, ctx->pinned.reserve(bytes));
    SFM_CUDA(ctx, ctx->scratch.reserve(bytes));
    Carver hc(ctx->pinned.p);
    float* h_pts = hc.take<float>(2 * (size_t)NP);
    int32_t* h_mq = hc.take<int32_t>((size_t)M);
    int32_t* h_mt = hc.take<int32_t>((size_t)M);
    int32_t* h_nk = hc.take<int32_t>(n_pairs);
    float* h_X = hc.take<float>(3 * (size_t)M);
    uint8_t* h_keep = hc.take<uint8_t>((size_t)M);
    const size_t up_len = (char*)(h_nk + n_pairs) - (char*)ctx->pinned.p;
    const size_t down_off = (char*)h_nk - (char*)ctx->pinned.p, down_len = hc.off - down_off;
    if (NP > 0) memcpy(h_pts, pts, 8 * (size_t)NP);
    memcpy(h_mq, match_q, 4 * (size_t)M);
    memcpy(h_mt, match_t, 4 * (size_t)M);
    memset(h_nk, 0, 4 * (size_t)n_pairs);
    Carver cv(ctx->scratch.p);
    const float2* d_pts = (const float2*)cv.take<float>(2 * (size_t)NP);
    const int32_t* d_mq = cv.take<int32_t>((size_t)M);
    const int32_t* d_mt = cv.take<int32_t>((size_t)M);
    int32_t* d_nk = cv.take<int32_t>(n_pairs);
    float* d_X = cv.take<float>(3 * (size_t)M);
    uint8_t* d_keep = cv.take<uint8_t>((size_t)M);
    SFM_CUDA(ctx, cudaMemcpyAsync(ctx->scratch.p, ctx->pinned.p, up_len, cudaMemcpyHostToDevice, ctx->stream));
    for (int p = 0; p < n_pairs; ++p) {
        const int64_t off = match_off[p];
        const int m = (int)(match_off[p + 1] - off);
        if (m == 0) continue;
        TriParams P; make_params(K, poses + 24 * (size_t)p, poses + 24 * (size_t)p + 12, max_reproj_px, P);
        triangulate_kernel<<<ceil_div(m, 128), 128, 0, ctx->stream>>>(P, d_pts + img_off[pairs[2 * p]], d_pts + img_off[pairs[2 * p + 1]],
                                                                      d_mq + off, d_mt + off, m, d_X + 3 * off, d_keep + off, d_nk + p);
        SFM_LAUNCH_CHECK(ctx);
    }
    SFM_CUDA(ctx, cudaMemcpyAsync((char*)ctx->pinned.p + down_off, (char*)ctx->scratch.p + down_off, down_len, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(X, h_X, 12 * (size_t)M);
    memcpy(keep, h_keep, (size_t)M);
    if (n_keep) memcpy(n_keep, h_nk, 4 * (size_t)n_pairs);
    return SFMB200_OK;
}

}  // extern "C"
