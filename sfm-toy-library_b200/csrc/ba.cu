// ba.cu -- K3/K4: bundle adjustment as Levenberg-Marquardt with per-point Schur elimination, all on the device.
//
// Replaces SfMBundleAdjustmentUtils::adjustBundle (reference SfMToyLib/SfMBundleAdjustmentUtils.cpp:99-222), i.e.
// ceres::Solve with LM + DENSE_SCHUR over AutoDiffCostFunction<SimpleReprojectionError,2,6,3,1> blocks (:58-97,
// :158-164, :171-179).  Ceres' algorithm is restated (SURVEY.md appendix A.3): Jacobi column scaling fixed at x0,
// LM diagonal clamp(diag(J^T J), 1e-6, 1e32)/radius, step-quality radius update, the four termination tests.
//
// Design (GPU-first, not a Ceres translation):
//   * The Jacobian is never materialised.  Every pass re-evaluates the closed-form 2x(6+3+1) blocks from 8-byte
//     observations (ba_math.cuh) -- HBM traffic per LM iteration is the observation list + the point/camera state.
//   * ba_point_kernel   (K3a, point-major, one sub-warp group per 3D point): U_p = sum Jp^T Jp + D_p^2, its Cholesky
//     inverse M_p, g_p, and per observation Z_o = Jc^T Jp M^T (Zbuf, 144 bytes per observation).
//   * ba_pair_kernel    (K3c, ba_row.cuh): the off-diagonal blocks  S[ci,cj] -= sum Z_i Z_j^T  from per-(camera pair, point
//     segment) entry lists sorted by point, one mma.sync.m8n8k4.f64 per entry, one partial block per (pair, segment, split).
//   * ba_camera_kernel<DET> (camera-major slices of the stable camera-sorted list): diagonal blocks, camera-focal column, rhs,
//     gradient and J^T J diagonal, one partial record per (slice, camera).  ba_combine_kernel sums the partial blocks and
//     records in a fixed order: no floating-point atomics, bitwise reproducible.
//     ("red" mode, SFMB200_BA_SCHUR=red or more cameras than the partial buffers allow, keeps the per-point
//     red.global.add.f64 formulation with the register-accumulating ba_camera_kernel.)
//   * reduced system summed over ranks: peer-memory kernel (loads the peers' buffers over NVLink into a local summed copy)
//     or one NCCL all-reduce (S, rhs, gradient, diag, cost in one buffer).
//   * ba_assemble + chol.cuh (streaming dataflow tile Cholesky, rhs carried as an extra row so the forward substitution is
//     free, back substitution with inverse diagonal tiles on a CTA cluster or, for large n, one CTA): K4.
//   * ba_backsub_eval_kernel (point-major, default): delta_p from Jacobians re-evaluated at x, candidate point, model cost
//     change and candidate cost fused; ba_backsub_z_kernel (SFMB200_BA_BACKSUB=stored) reads the stored Z blocks instead.
//   LM control runs on the DEVICE (LMState, ba_lm_control_kernel); the host enqueues chunks of iterations and reads the
//   state back once per chunk.
#include "common.cuh"
#include "ba_math.cuh"
#include "chol.cuh"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>

namespace {

constexpr int PT_THREADS = 128;
constexpr int PTB = 18;                // doubles per point in ptblk
constexpr int CAM_THREADS = 128;

// Levenberg-Marquardt control state, resident on the device: the kernels of an iteration read `cur` (which of the two
// state buffers is x), `radius` and `status` from it, ba_lm_control_kernel updates it after every iteration, and the host
// only reads it back once per chunk of iterations (no stream sync per iteration).
struct LMState {
    double radius, decrease_factor, x_cost, x_norm, gmax, initial_cost;
    double msg_a, msg_b;              // numbers quoted in the termination message
    double last_rho;
    int cur, iter, invalid_steps, new_point;
    int status;                       // 0 = running; otherwise LM_* reason, every later kernel of the chunk is a no-op
    int termination_type;
    int num_successful, num_unsuccessful;
    int passes;                       // iterations whose kernels actually ran
};
enum { LM_RUNNING = 0, LM_EVAL_FAILED = 1, LM_GRADIENT_TOL = 2, LM_MAX_TIME = 3, LM_MAX_ITER = 4, LM_MIN_RADIUS = 5, LM_INVALID_STEPS = 6,
       LM_PARAMETER_TOL = 7, LM_FUNCTION_TOL = 8 };

struct BAView {
    int nc, np, nobs, maxk;
    // device-resident LM loop (st != nullptr): both state buffers; the kernels pick x = buffer st->cur themselves
    const LMState* st;
    double* cf2[2]; double* pts2[2]; CamDerived* camd2[2];
    // point-major observations
    const float2* obs_xy; const int32_t* obs_cam; const int32_t* pt_off;
    // camera-major copy
    const int32_t* cm_off; const float2* cm_xy; const int32_t* cm_pt;
    // state
    const double* cams; const double* pts; const double* focal;      // current x (focal = cams + 6*nc)
    const CamDerived* camd;                                           // derived per camera at x
    const double* scale_cf; const double* scale_pt;                   // Jacobi scaling
    double* ptblk;                                                    // [np*PTB] M(6) zg(3) zf(3) g(3) diag(U)(3)
    double* Zbuf;                                                     // [nobs*18] Z_o = Jc^T Jp M^T (gather mode), point-major
    // reduced system (block layout) + sums
    double* Sblk; double* Scf; double* Sff; double* rhs; double* gcf; double* dcf; double* sums;
    unsigned long long* gmax_pt_bits;                                 // max |g_p| (bit pattern of a non-negative double)
    int* fail;                                                        // count of non-SPD point blocks
    double min_diag, max_diag;
    double* part4;                                                    // [grid][4] per-CTA partial sums of the point-major kernels (row mode)
    unsigned* counters;                                               // [0] point kernel, [1] back-substitution, [2] combine: "last CTA" tickets
};

// Fixed-order reduction of per-CTA partial sums by the LAST CTA to finish (whoever that is, the order of the additions is the
// same): every CTA stores its 4 partials, takes a ticket; the last one lets warp 0 add partials lane, lane+32, ... and then a
// fixed shuffle tree.  Returns true in the threads of warp 0 of the last CTA, with the totals in out[0..3].  The ticket
// counter wraps to zero, ready for the next launch.
__device__ __forceinline__ bool last_block_sum4(double* __restrict__ part4, unsigned* __restrict__ counter, const double (&mine)[4], double (&out)[4]) {
    __shared__ bool last_s;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) part4[4 * (size_t)blockIdx.x + q] = mine[q];
        __threadfence();
        last_s = atomicInc(counter, gridDim.x - 1) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last_s || threadIdx.x >= 32) return false;
    __threadfence();
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (unsigned b = threadIdx.x; b < gridDim.x; b += 32) {
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] += __ldcg(part4 + 4 * (size_t)b + q);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
        out[q] = acc[q];
    }
    return true;
}

// The current x of a kernel: the view's own pointers, or -- inside an LM chunk -- buffer st->cur.  run = false when the solve
// has already terminated (the kernel is a no-op).  (Kept out of BAView: writing to the by-value parameter struct makes the
// compiler copy all of it to local memory.)
struct LMX { const double* focal; const double* pts; const CamDerived* camd; bool run; };
__device__ __forceinline__ LMX lm_x(const BAView& v) {
    LMX x; x.focal = v.focal; x.pts = v.pts; x.camd = v.camd; x.run = true;
    if (v.st) {
        x.run = v.st->status == LM_RUNNING;
        const int cur = v.st->cur;
        x.focal = v.cf2[cur] + 6 * v.nc; x.pts = v.pts2[cur]; x.camd = v.camd2[cur];
    }
    return x;
}

__device__ __forceinline__ void red_add(double* p, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ double clampd(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }
__device__ __forceinline__ size_t blk_index(int i, int j, int nb) {   // i <= j
    return (size_t)i * nb - (size_t)i * (i - 1) / 2 + (j - i);
}

template <int G>
__device__ __forceinline__ double group_sum(double v, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// scaled Jacobian blocks of one observation
struct ObsJ { double r[2], Jc[12], Jp[6], Jf[2]; };
__device__ __forceinline__ void eval_scaled(const CamDerived& d, const double* X, double f, float2 xy,
                                            const double* sc /*6*/, const double* sp /*3*/, double sf, ObsJ& o) {
    obs_eval(d, X, f, (double)xy.x, (double)xy.y, o.r, o.Jc, o.Jp, o.Jf);
#pragma unroll
    for (int a = 0; a < 6; ++a) { o.Jc[a] *= sc[a]; o.Jc[6 + a] *= sc[a]; }
#pragma unroll
    for (int a = 0; a < 3; ++a) { o.Jp[a] *= sp[a]; o.Jp[3 + a] *= sp[a]; }
    o.Jf[0] *= sf; o.Jf[1] *= sf;
}

__global__ void cam_derive_kernel(const double* __restrict__ cams, int nc, CamDerived* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < nc) { CamDerived d; cam_derive(cams + 6 * c, d); out[c] = d; }
}

// ---------------------------------------------------------------------------------------------------------------
// Jacobi scaling (computed once at x0): squared column norms of the UNSCALED Jacobian.
// points: scale_pt written directly; cameras/focal: accumulated into colnorm_cf (summed over ranks afterwards).
// ---------------------------------------------------------------------------------------------------------------
template <int G>
__global__ void __launch_bounds__(PT_THREADS) ba_point_norm_kernel(BAView v, double* __restrict__ scale_pt_out) {
    const int lane = threadIdx.x & 31, gl = lane % G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << ((lane / G) * G));
    const int groups_per_block = PT_THREADS / G;
    const double f = *v.focal;
    for (int p = blockIdx.x * groups_per_block + threadIdx.x / G; p < v.np; p += gridDim.x * groups_per_block) {
        const int o0 = v.pt_off[p], k = v.pt_off[p + 1] - o0;
        const double X[3] = {v.pts[3 * p], v.pts[3 * p + 1], v.pts[3 * p + 2]};
        double n0 = 0, n1 = 0, n2 = 0;
        for (int j = gl; j < k; j += G) {
            const int o = o0 + j;
            double r[2], Jc[12], Jp[6], Jf[2];
            const float2 xy = v.obs_xy[o];
            obs_eval(v.camd[v.obs_cam[o]], X, f, (double)xy.x, (double)xy.y, r, Jc, Jp, Jf);
            n0 += Jp[0] * Jp[0] + Jp[3] * Jp[3]; n1 += Jp[1] * Jp[1] + Jp[4] * Jp[4]; n2 += Jp[2] * Jp[2] + Jp[5] * Jp[5];
        }
        n0 = group_sum<G>(n0, gmask); n1 = group_sum<G>(n1, gmask); n2 = group_sum<G>(n2, gmask);
        if (gl == 0) {
            scale_pt_out[3 * p] = 1.0 / (1.0 + sqrt(n0)); scale_pt_out[3 * p + 1] = 1.0 / (1.0 + sqrt(n1));
            scale_pt_out[3 * p + 2] = 1.0 / (1.0 + sqrt(n2));
        }
    }
}

__global__ void __launch_bounds__(CAM_THREADS) ba_camera_norm_kernel(BAView v, double* __restrict__ colnorm_cf) {
    const int c = blockIdx.y;
    const int begin = v.cm_off[c], end = v.cm_off[c + 1];
    const CamDerived d = v.camd[c];
    const double f = *v.focal;
    double n[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int i = begin + blockIdx.x * CAM_THREADS + threadIdx.x; i < end; i += gridDim.x * CAM_THREADS) {
        const int p = v.cm_pt[i];
        const double X[3] = {v.pts[3 * p], v.pts[3 * p + 1], v.pts[3 * p + 2]};
        double r[2], Jc[12], Jp[6], Jf[2];
        const float2 xy = v.cm_xy[i];
        obs_eval(d, X, f, (double)xy.x, (double)xy.y, r, Jc, Jp, Jf);
#pragma unroll
        for (int a = 0; a < 6; ++a) n[a] += Jc[a] * Jc[a] + Jc[6 + a] * Jc[6 + a];
        n[6] += Jf[0] * Jf[0] + Jf[1] * Jf[1];
    }
    __shared__ double red[CAM_THREADS / 32][7];
#pragma unroll
    for (int a = 0; a < 7; ++a) { const double s = warp_sum(n[a]); if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][a] = s; }
    __syncthreads();
    if (threadIdx.x < 7) {
        double s = 0;
        for (int w = 0; w < CAM_THREADS / 32; ++w) s += red[w][threadIdx.x];
        if (s != 0.0) red_add(threadIdx.x < 6 ? colnorm_cf + 6 * c + threadIdx.x : colnorm_cf + 6 * v.nc, s);
    }
}

__global__ void scale_from_norm_kernel(const double* __restrict__ colnorm, int n, double* __restrict__ scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) scale[i] = 1.0 / (1.0 + sqrt(colnorm[i]));
}
__global__ void fill_kernel(double* __restrict__ p, size_t n, double v) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ---------------------------------------------------------------------------------------------------------------
// K3a: point-major elimination.  One group of G lanes per 3D point (G = 4/8/16/32 >= observations per point when
// possible); lanes evaluate the point's observations in parallel, group-reduce U_p / g_p with warp shuffles, and the
// whole warp then sweeps the pair blocks of each of its points so that 32 consecutive doubles go out per RED.
// Shared memory per group: Z [maxk][18] + camera ids [maxk]; pair table shared by the CTA.
// ---------------------------------------------------------------------------------------------------------------
template <int G, bool GATHER>
__global__ void __launch_bounds__(PT_THREADS, 3) ba_point_kernel(BAView v, double inv_radius) {
    const LMX x = lm_x(v);
    if (!x.run) return;
    if (v.st) inv_radius = 1.0 / v.st->radius;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ __align__(16) double zstage[GATHER ? PT_THREADS / 32 : 1][GATHER ? 32 * 18 : 2];      // one warp-iteration of Z records
    constexpr int GB = PT_THREADS / G, GW = 32 / G;
    const int maxk = v.maxk;
    double* Zall = reinterpret_cast<double*>(smem_raw);                           // [GB][maxk][18]   (RED mode only)
    int* camall = reinterpret_cast<int*>(Zall + (size_t)GB * maxk * 18);          // [GB][maxk]
    unsigned short* pair_tab = reinterpret_cast<unsigned short*>(camall + GB * maxk);   // [maxk*(maxk-1)/2]  (i | j<<8)
    if (!GATHER) {
        for (int j = 1 + threadIdx.x / 32; j < maxk; j += PT_THREADS / 32)
            for (int i = threadIdx.x & 31; i < j; i += 32) pair_tab[j * (j - 1) / 2 + i] = (unsigned short)(i | (j << 8));
        __syncthreads();
    }

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gl = lane % G, gi = lane / G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
    const int group_in_block = warp * GW + gi;
    double* Zg = GATHER ? nullptr : Zall + (size_t)group_in_block * maxk * 18;
    int* camg = GATHER ? nullptr : camall + group_in_block * maxk;
    const double f = *x.focal, sf = v.scale_cf[6 * v.nc];
    const int nb = v.nc;

    double acc_cost = 0, acc_xn = 0, acc_sff = 0, acc_rf = 0, acc_gmax = 0;
    const int np_round = (v.np + GB - 1) / GB * GB;
    for (int base = blockIdx.x * GB; base < np_round; base += gridDim.x * GB) {
        const int p = base + group_in_block;
        const bool active = p < v.np;
        int o0 = 0, k = 0;
        double X[3] = {0, 0, 0}, sp[3] = {1, 1, 1};
        {   // pull the next iteration's point and observation lines into L2 while this one computes (no registers held)
            const int pn = p + gridDim.x * GB;
            if (pn < v.np && gl == 0) {
                const int on = v.pt_off[pn];
                asm volatile("prefetch.global.L2 [%0];" :: "l"(v.obs_cam + on)); asm volatile("prefetch.global.L2 [%0];" :: "l"(v.obs_xy + on));
                asm volatile("prefetch.global.L2 [%0];" :: "l"(x.pts + 3 * (size_t)pn)); asm volatile("prefetch.global.L2 [%0];" :: "l"(v.scale_pt + 3 * (size_t)pn));
            }
        }
        if (active) {
            o0 = v.pt_off[p]; k = v.pt_off[p + 1] - o0;
            X[0] = x.pts[3 * p]; X[1] = x.pts[3 * p + 1]; X[2] = x.pts[3 * p + 2];
            sp[0] = v.scale_pt[3 * p]; sp[1] = v.scale_pt[3 * p + 1]; sp[2] = v.scale_pt[3 * p + 2];
        }
        double U[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0}, wf[3] = {0, 0, 0}, cost = 0;
        double Wreg[18];                  // gather mode: W of this lane's first observation stays in registers
        for (int j = gl; j < k; j += G) {
            const int o = o0 + j, c = v.obs_cam[o];
            ObsJ J;
            eval_scaled(x.camd[c], X, f, v.obs_xy[o], v.scale_cf + 6 * c, sp, sf, J);
            const double* e = J.Jp;
            U[0] += e[0] * e[0] + e[3] * e[3]; U[1] += e[0] * e[1] + e[3] * e[4]; U[2] += e[0] * e[2] + e[3] * e[5];
            U[3] += e[1] * e[1] + e[4] * e[4]; U[4] += e[1] * e[2] + e[4] * e[5]; U[5] += e[2] * e[2] + e[5] * e[5];
#pragma unroll
            for (int a = 0; a < 3; ++a) { g[a] += e[a] * J.r[0] + e[3 + a] * J.r[1]; wf[a] += e[a] * J.Jf[0] + e[3 + a] * J.Jf[1]; }
            cost += J.r[0] * J.r[0] + J.r[1] * J.r[1];
            // W = Jc^T Jp (6x3), turned into Z = W M^T below
            if (GATHER && j == gl) {
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b) Wreg[a * 3 + b] = J.Jc[a] * e[b] + J.Jc[6 + a] * e[3 + b];
            } else {
                double* W = GATHER ? v.Zbuf + (size_t)o * 18 : Zg + j * 18;
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b) W[a * 3 + b] = J.Jc[a] * e[b] + J.Jc[6 + a] * e[3 + b];
            }
            if (!GATHER) camg[j] = c;
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) U[a] = group_sum<G>(U[a], gmask);
#pragma unroll
        for (int a = 0; a < 3; ++a) { g[a] = group_sum<G>(g[a], gmask); wf[a] = group_sum<G>(wf[a], gmask); }
        cost = group_sum<G>(cost, gmask);

        const double udiag[3] = {U[0], U[3], U[5]};                  // diag(J_p^T J_p), kept for the model cost (back-substitution kernel)
        // LM diagonal of the point block: clamp(diag(J^T J)) / radius
        U[0] += clampd(U[0], v.min_diag, v.max_diag) * inv_radius;
        U[3] += clampd(U[3], v.min_diag, v.max_diag) * inv_radius;
        U[5] += clampd(U[5], v.min_diag, v.max_diag) * inv_radius;
        double M[6] = {0, 0, 0, 0, 0, 0};
        const bool ok = chol3_inverse(U, M);
        if (!ok) { M[0] = M[1] = M[2] = M[3] = M[4] = M[5] = 0.0; }
        // zg = M g, zf = M wf
        const double zg[3] = {M[0] * g[0], M[1] * g[0] + M[2] * g[1], M[3] * g[0] + M[4] * g[1] + M[5] * g[2]};
        const double zf[3] = {M[0] * wf[0], M[1] * wf[0] + M[2] * wf[1], M[3] * wf[0] + M[4] * wf[1] + M[5] * wf[2]};
        if (active) {
            const double blk[PTB] = {M[0], M[1], M[2], M[3], M[4], M[5], zg[0], zg[1], zg[2], zf[0], zf[1], zf[2], g[0], g[1], g[2], udiag[0], udiag[1], udiag[2]};
#pragma unroll
            for (int q = 0; q < PTB; ++q) if ((q % G) == gl) v.ptblk[(size_t)p * PTB + q] = blk[q];
            if (gl == 0) {
                if (!ok && k > 0) atomicAdd(v.fail, 1);
                acc_cost += cost;
                acc_xn += X[0] * X[0] + X[1] * X[1] + X[2] * X[2];
                acc_sff += zf[0] * zf[0] + zf[1] * zf[1] + zf[2] * zf[2];
                acc_rf += zf[0] * zg[0] + zf[1] * zg[1] + zf[2] * zg[2];
                acc_gmax = fmax(acc_gmax, fmax(fabs(g[0] / sp[0]), fmax(fabs(g[1] / sp[1]), fabs(g[2] / sp[2]))));
            }
        }
        // Z = W M^T  (own rows; same thread wrote W).  A lane-per-record store touches 36 cache lines per instruction (records
        // are 144 bytes apart): with at most G observations per point the warp's records are one contiguous range of Zbuf, so
        // they are assembled in shared memory (16-byte stores at a 36-word lane stride are conflict free) and written out with
        // fully coalesced 16-byte stores.
        const bool stage = GATHER && v.maxk <= G;
        int o_first = 0, o_end = 0;
        if (stage) {
            const int p_first = base + warp * GW;
            o_first = p_first < v.np ? v.pt_off[p_first] : 0; o_end = p_first < v.np ? v.pt_off[min(p_first + GW, v.np)] : 0;
        }
        if (GATHER && gl < k) {
            double2* dst = stage ? reinterpret_cast<double2*>(zstage[warp] + (size_t)(o0 + gl - o_first) * 18)
                                 : reinterpret_cast<double2*>(v.Zbuf + (size_t)(o0 + gl) * 18);
#pragma unroll
            for (int a = 0; a < 6; a += 2) {      // two rows = six doubles = three 16-byte stores
                double z[6];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const double w0 = Wreg[(a + h) * 3], w1 = Wreg[(a + h) * 3 + 1], w2 = Wreg[(a + h) * 3 + 2];
                    z[3 * h] = w0 * M[0]; z[3 * h + 1] = w0 * M[1] + w1 * M[2]; z[3 * h + 2] = w0 * M[3] + w1 * M[4] + w2 * M[5];
                }
                dst[a / 2 * 3] = make_double2(z[0], z[1]); dst[a / 2 * 3 + 1] = make_double2(z[2], z[3]); dst[a / 2 * 3 + 2] = make_double2(z[4], z[5]);
            }
        }
        if (stage) {
            __syncwarp();
            const double2* src = reinterpret_cast<const double2*>(zstage[warp]);
            double2* out = reinterpret_cast<double2*>(v.Zbuf + (size_t)o_first * 18);
            for (int i = lane; i < (o_end - o_first) * 9; i += 32) out[i] = src[i];
            __syncwarp();
        }
        for (int j = gl + (GATHER ? G : 0); j < k; j += G) {
            double* W = GATHER ? v.Zbuf + (size_t)(o0 + j) * 18 : Zg + j * 18;
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                const double w0 = W[a * 3], w1 = W[a * 3 + 1], w2 = W[a * 3 + 2];
                W[a * 3] = w0 * M[0]; W[a * 3 + 1] = w0 * M[1] + w1 * M[2]; W[a * 3 + 2] = w0 * M[3] + w1 * M[4] + w2 * M[5];
            }
        }
        if (GATHER) continue;           // off-diagonal blocks are accumulated by ba_pair_kernel from Zbuf
        __syncwarp();
        // pair sweep: the whole warp handles the points of its GW groups one after the other
#pragma unroll 1
        for (int gs = 0; gs < GW; ++gs) {
            const int kk = __shfl_sync(0xffffffffu, k, gs * G);
            const double* Zs = Zall + (size_t)(warp * GW + gs) * maxk * 18;
            const int* cs = camall + (warp * GW + gs) * maxk;
            const int total = kk * (kk - 1) / 2 * 36;
            for (int e = lane; e < total; e += 32) {
                const int pr = e / 36, ab = e - pr * 36, a = ab / 6, b = ab - a * 6;
                const unsigned ij = pair_tab[pr];
                const int i = ij & 0xff, j = ij >> 8;
                const double* zi = Zs + i * 18 + a * 3; const double* zj = Zs + j * 18 + b * 3;
                const double val = zi[0] * zj[0] + zi[1] * zj[1] + zi[2] * zj[2];
                red_add(v.Sblk + blk_index(cs[i], cs[j], nb) * 36 + ab, -val);
            }
        }
        __syncwarp();
    }
    // CTA reduction of the scalar accumulators
    __shared__ double sred[PT_THREADS / 32][5];
    const double c0 = warp_sum(acc_cost), c1 = warp_sum(acc_xn), c2 = warp_sum(acc_sff), c3 = warp_sum(acc_rf), c4 = warp_max(acc_gmax);
    if (lane == 0) { sred[warp][0] = c0; sred[warp][1] = c1; sred[warp][2] = c2; sred[warp][3] = c3; sred[warp][4] = c4; }
    __syncthreads();
    double t[4] = {0, 0, 0, 0};
    if (threadIdx.x == 0) {
        double t4 = 0;
        for (int w = 0; w < PT_THREADS / 32; ++w) { t[0] += sred[w][0]; t[1] += sred[w][1]; t[2] += sred[w][2]; t[3] += sred[w][3]; t4 = fmax(t4, sred[w][4]); }
        atomicMax(v.gmax_pt_bits, (unsigned long long)__double_as_longlong(t4));     // a maximum: order-independent
        if (!GATHER) {                                                               // "red" mode: accumulating atomics
            red_add(v.sums + 0, t[0]); red_add(v.sums + 1, t[1]);
            red_add(v.Sff, -t[2]); red_add(v.rhs + 6 * v.nc, -t[3]);
        }
    }
    if (GATHER) {                      // row mode: fixed-order sum by the last CTA; plain stores (ba_combine_kernel adds the camera part)
        double tot[4];
        if (last_block_sum4(v.part4, v.counters + 0, t, tot) && threadIdx.x == 0) {
            v.sums[0] = tot[0]; v.sums[1] = tot[1]; *v.Sff = -tot[2]; v.rhs[6 * v.nc] = -tot[3];
        }
    }
}

// one FP64 tensor-core product: D(8x8) += A(8x4) B(4x8); lane l holds A[l>>2][l&3], B[l&3][l>>2], D[l>>2][2(l&3)], D[l>>2][2(l&3)+1]
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// ---------------------------------------------------------------------------------------------------------------
// K3b (DET = false in "red" mode; DET = true in gather mode, summed by ba_combine_kernel): camera-major pass over the camera-sorted observation list.  Every CTA takes an equal, contiguous slice of the list
// (grid = number of co-resident CTAs, one balanced wave; a per-camera grid left a third of the run to a ragged last wave)
// and walks the cameras its slice touches.  Per camera: diagonal block, camera-focal column, rhs, gradient and J^T J
// diagonal, all in registers; one reduction per (CTA, camera).
// ---------------------------------------------------------------------------------------------------------------
// DET: instead of accumulating into the reduced system with atomics, every (slice, camera) segment stores ONE partial record
// (cam_part[(slice + camera)][CAM_REC]); ba_combine_kernel adds the records of a camera in slice order (row mode: bitwise
// reproducible).  NORM_ONLY (DET only): just the squared column norms of the UNSCALED Jacobian (Jacobi scaling at x0).
constexpr int CAM_REC = 64;      // [0,36) diagonal block (full), [36,42) camera-focal, [42,48) rhs, [48,54) gradient, [54,60) diag J^T J, 60 Jf^T Jf, 61 Jf^T r
template <bool DET, bool NORM_ONLY>
__global__ void __launch_bounds__(CAM_THREADS) ba_camera_kernel(BAView v, int per_cta, double* __restrict__ cam_part) {
    const LMX x = lm_x(v);
    if (!x.run) return;
    const int start = blockIdx.x * per_cta, stop = min(v.nobs, start + per_cta);
    if (start >= stop) return;
    int c = 0;
    {   // last camera whose list begins at or before `start`
        int lo = 0, hi = v.nc - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (v.cm_off[mid] <= start) lo = mid; else hi = mid - 1; }
        c = lo;
    }
    const double f = *x.focal, sf = NORM_ONLY ? 1.0 : v.scale_cf[6 * v.nc];
    __shared__ double red[CAM_THREADS / 32][48];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (; c < v.nc && v.cm_off[c] < stop; ++c) {
    const int begin = max(start, v.cm_off[c]), end = min(stop, v.cm_off[c + 1]);
    if (begin >= end) continue;
    const CamDerived d = x.camd[c];
    double sc[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) sc[a] = NORM_ONLY ? 1.0 : v.scale_cf[6 * c + a];
    // accumulators: A[21] diag block (upper), C[6] cam-focal, R[6] rhs, Gd[6] gradient, D[6] diag, ff, gf
    double A[21], Cf[6], R[6], Gd[6], D[6], ff = 0, gf = 0;
#pragma unroll
    for (int a = 0; a < 21; ++a) A[a] = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) { Cf[a] = 0; R[a] = 0; Gd[a] = 0; D[a] = 0; }
    for (int i = begin + threadIdx.x; i < end; i += CAM_THREADS) {
        const int p = v.cm_pt[i];
        const double X[3] = {x.pts[3 * p], x.pts[3 * p + 1], x.pts[3 * p + 2]};
        ObsJ J;
        if (NORM_ONLY) {
            const double one[3] = {1.0, 1.0, 1.0};
            eval_scaled(d, X, f, v.cm_xy[i], sc, one, 1.0, J);
            ff += J.Jf[0] * J.Jf[0] + J.Jf[1] * J.Jf[1];
#pragma unroll
            for (int a = 0; a < 6; ++a) D[a] += J.Jc[a] * J.Jc[a] + J.Jc[6 + a] * J.Jc[6 + a];
            continue;
        }
        const double sp[3] = {v.scale_pt[3 * p], v.scale_pt[3 * p + 1], v.scale_pt[3 * p + 2]};
        const double* pb = v.ptblk + (size_t)p * PTB;
        const double M[6] = {pb[0], pb[1], pb[2], pb[3], pb[4], pb[5]};
        const double zg[3] = {pb[6], pb[7], pb[8]}, zf[3] = {pb[9], pb[10], pb[11]};
        eval_scaled(d, X, f, v.cm_xy[i], sc, sp, sf, J);
        ff += J.Jf[0] * J.Jf[0] + J.Jf[1] * J.Jf[1];
        gf += J.Jf[0] * J.r[0] + J.Jf[1] * J.r[1];
        double Z[6][3];
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            const double w0 = J.Jc[a] * J.Jp[0] + J.Jc[6 + a] * J.Jp[3], w1 = J.Jc[a] * J.Jp[1] + J.Jc[6 + a] * J.Jp[4],
                         w2 = J.Jc[a] * J.Jp[2] + J.Jc[6 + a] * J.Jp[5];
            Z[a][0] = w0 * M[0]; Z[a][1] = w0 * M[1] + w1 * M[2]; Z[a][2] = w0 * M[3] + w1 * M[4] + w2 * M[5];
            const double jr = J.Jc[a] * J.r[0] + J.Jc[6 + a] * J.r[1];
            Gd[a] += jr;
            R[a] += jr - (Z[a][0] * zg[0] + Z[a][1] * zg[1] + Z[a][2] * zg[2]);
            Cf[a] += J.Jc[a] * J.Jf[0] + J.Jc[6 + a] * J.Jf[1] - (Z[a][0] * zf[0] + Z[a][1] * zf[1] + Z[a][2] * zf[2]);
            D[a] += J.Jc[a] * J.Jc[a] + J.Jc[6 + a] * J.Jc[6 + a];
        }
        int q = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = a; b < 6; ++b, ++q)
                A[q] += J.Jc[a] * J.Jc[b] + J.Jc[6 + a] * J.Jc[6 + b] - (Z[a][0] * Z[b][0] + Z[a][1] * Z[b][1] + Z[a][2] * Z[b][2]);
    }
    // CTA reduction: 47 values
#pragma unroll
    for (int a = 0; a < 21; ++a) { const double s = warp_sum(A[a]); if (lane == 0) red[warp][a] = s; }
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        const double s0 = warp_sum(Cf[a]), s1 = warp_sum(R[a]), s2 = warp_sum(Gd[a]), s3 = warp_sum(D[a]);
        if (lane == 0) { red[warp][21 + a] = s0; red[warp][27 + a] = s1; red[warp][33 + a] = s2; red[warp][39 + a] = s3; }
    }
    { const double s0 = warp_sum(ff), s1 = warp_sum(gf); if (lane == 0) { red[warp][45] = s0; red[warp][46] = s1; } }
    __syncthreads();
    if (threadIdx.x < 47) {
        double s = 0;
        for (int w = 0; w < CAM_THREADS / 32; ++w) s += red[w][threadIdx.x];
        const int t = threadIdx.x, fidx = 6 * v.nc;
        if (DET) {
            double* rec = cam_part + (size_t)(blockIdx.x + c) * CAM_REC;
            if (t < 21) {
                int a = 0, rem = t; while (rem >= 6 - a) { rem -= 6 - a; ++a; } const int b = a + rem;
                rec[a * 6 + b] = s; rec[b * 6 + a] = s;
            } else rec[36 + (t - 21)] = s;           // 21..26 -> 36..41, 27..32 -> 42..47, 33..38 -> 48..53, 39..44 -> 54..59, 45 -> 60, 46 -> 61
        } else if (t < 21) {
            // upper-triangular index t -> (a,b); write both halves of the (symmetric) diagonal block
            int a = 0, rem = t; while (rem >= 6 - a) { rem -= 6 - a; ++a; } const int b = a + rem;
            double* blk = v.Sblk + blk_index(c, c, v.nc) * 36;
            red_add(blk + a * 6 + b, s);
            if (a != b) red_add(blk + b * 6 + a, s);
        } else if (t < 27) red_add(v.Scf + 6 * c + (t - 21), s);
        else if (t < 33) red_add(v.rhs + 6 * c + (t - 27), s);
        else if (t < 39) red_add(v.gcf + 6 * c + (t - 33), s);
        else if (t < 45) red_add(v.dcf + 6 * c + (t - 39), s);
        else if (t == 45) { red_add(v.Sff, s); red_add(v.dcf + fidx, s); }
        else { red_add(v.rhs + fidx, s); red_add(v.gcf + fidx, s); }
    }
    __syncthreads();            // red[] is reused by the next camera of this slice
    }
}

#include "ba_row.cuh"

// ---------------------------------------------------------------------------------------------------------------
// K4: dense reduced system.  A is (npad x npad) row-major, lower triangle used, npad = multiple of NB > n;
// row n carries the right-hand side (forward substitution for free), remaining pad rows are identity.
// ---------------------------------------------------------------------------------------------------------------
__global__ void ba_assemble_kernel(const double* __restrict__ Sblk, const double* __restrict__ Scf, const double* __restrict__ Sff,
                                   const double* __restrict__ rhs, const double* __restrict__ dcf, int nc, int npad,
                                   double inv_radius, double min_diag, double max_diag, double* __restrict__ A, const LMState* __restrict__ st,
                                   unsigned* __restrict__ solve_counter) {
    if (st) { if (st->status != LM_RUNNING) return; inv_radius = 1.0 / st->radius; }
    // number of the dense solve that follows (the dataflow Cholesky's flags carry it): kept on the device so that a replayed
    // CUDA graph, whose kernel arguments are frozen, still sees a new number every time
    if (solve_counter && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *solve_counter += 1u;
    const int n = 6 * nc + 1;
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= npad || c > r) return;
    double val;
    if (r < n) {
        if (r == n - 1) val = (c == n - 1) ? *Sff : Scf[c];
        else {
            const int bi = r / 6, a = r - 6 * bi, bj = c / 6, b = c - 6 * bj;      // bj <= bi
            val = Sblk[blk_index(bj, bi, nc) * 36 + b * 6 + a];
        }
        if (r == c) val += clampd(dcf[r], min_diag, max_diag) * inv_radius;
    } else if (r == n) val = c < n ? rhs[c] : 0.0;          // augmented row (its own pivot is forced to 1)
    else val = (r == c) ? 1.0 : 0.0;
    A[(size_t)r * npad + c] = val;
}

// cameras + focal: candidate = x - y*scale ; derived table of the candidate ; norms.  Single CTA.
// locals[0] = |delta_cf|^2, [1] = |x_cf|^2, [2] = |cand_cf|^2, [3] = max |g_cf| (unscaled), [4] = camera part of -model cost change; post[7] = max |g_pts| (max-reduced over ranks)
__global__ void __launch_bounds__(256) ba_cam_update_kernel(BAView v, double inv_radius, const double* x_cf, const double* __restrict__ y_cf,
                                                            const double* __restrict__ scale_cf, const double* __restrict__ gcf, int nc,
                                                            double* cand_cf, CamDerived* camd_c, double* __restrict__ locals,
                                                            double* __restrict__ post, const unsigned long long* __restrict__ gmax_pt_bits,
                                                            const int* __restrict__ fail) {
    if (v.st) {                                 // device-resident LM loop: x = buffer cur, candidate = the other one
        if (v.st->status != LM_RUNNING) return;
        const int cur = v.st->cur;
        x_cf = v.cf2[cur]; cand_cf = v.cf2[cur ^ 1]; camd_c = v.camd2[cur ^ 1];
        inv_radius = 1.0 / v.st->radius;
    }
    const int n = 6 * nc + 1;
    double dn = 0, xn = 0, cn = 0, gm = 0, mc = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double yi = y_cf[i], d = -yi * scale_cf[i], xv = x_cf[i], cv = xv + d;
        cand_cf[i] = cv;
        const double dd = xv - cv;
        dn += dd * dd; xn += xv * xv; cn += cv * cv;
        gm = fmax(gm, fabs(gcf[i] / scale_cf[i]));
        // camera/focal part of the model cost change  1/2 y.(g + D^2 y)  (see ba_backsub_z_kernel), negated like post[1]
        mc -= 0.5 * yi * (gcf[i] + clampd(v.dcf[i], v.min_diag, v.max_diag) * inv_radius * yi);
    }
    __shared__ double red[8][5];
    const double a = warp_sum(dn), b = warp_sum(xn), c = warp_sum(cn), g = warp_max(gm), m = warp_sum(mc);
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = a; red[threadIdx.x >> 5][1] = b; red[threadIdx.x >> 5][2] = c; red[threadIdx.x >> 5][3] = g; red[threadIdx.x >> 5][4] = m; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
        for (int w = 0; w < 8; ++w) { s0 += red[w][0]; s1 += red[w][1]; s2 += red[w][2]; s3 = fmax(s3, red[w][3]); s4 += red[w][4]; }
        locals[0] = s0; locals[1] = s1; locals[2] = s2; locals[3] = s3; locals[4] = s4;
        // rank-local flags -> buffers that are reduced over ranks (sum / max) so that every rank takes the same decision
        post[7] = __longlong_as_double((long long)*gmax_pt_bits);      // max-reduced over ranks
        post[4] = (double)fail[0]; post[5] = (double)fail[1];
        post[0] = post[1] = post[2] = post[3] = post[6] = 0.0;        // accumulated by the back-substitution kernel that follows (not part of the pass memset: peers may still read it there)
    }
    __syncthreads();            // cand_cf complete
    for (int c2 = threadIdx.x; c2 < nc; c2 += blockDim.x) { CamDerived d; cam_derive(cand_cf + 6 * c2, d); camd_c[c2] = d; }
}

// ---------------------------------------------------------------------------------------------------------------
// LM control, one thread, after every iteration's evaluation: Ceres' TrustRegionMinimizer decisions (SURVEY.md appendix
// A.3; order of the tests: gradient, radius, [iteration], invalid step, parameter tolerance, function tolerance, step
// quality) on the scalars the kernels left in sums[8] | post[8] | locals[8].  Same arithmetic as a host loop would do;
// all ranks hold identical inputs (post and sums are rank-reduced), so every rank takes the same decision.
// ---------------------------------------------------------------------------------------------------------------
__global__ void ba_lm_control_kernel(LMState* __restrict__ st, const double* __restrict__ sums, const double* __restrict__ post,
                                     const double* __restrict__ locals, sfmb200_ba_options opt) {
    if (threadIdx.x != 0 || blockIdx.x != 0 || st->status != LM_RUNNING) return;
    LMState s = *st;
    ++s.passes;
    const double cost_x = 0.5 * sums[0], xn2_pts = sums[1];
    const double cand_cost_raw = 0.5 * post[0], model_acc = post[1] + locals[4], dn2_pts = post[2], cn2_pts = post[3];
    const double fail0 = post[4], fail1 = post[5], gmax_pt = post[7];
    const double dn2_cf = locals[0], xn2_cf = locals[1], cn2_cf = locals[2], gmax_cf = locals[3];
    auto stop = [&](int status, int type) { s.status = status; s.termination_type = type; *st = s; };
    if (s.new_point) {
        s.x_cost = cost_x; s.x_norm = sqrt(xn2_pts + xn2_cf); s.gmax = fmax(gmax_pt, gmax_cf);
        s.new_point = 0;
        if (s.iter == 0) {
            s.initial_cost = s.x_cost;
            if (!isfinite(s.x_cost)) return stop(LM_EVAL_FAILED, SFMB200_BA_FAILURE);
            if (s.gmax <= opt.gradient_tolerance) return stop(LM_GRADIENT_TOL, SFMB200_BA_CONVERGENCE);
            if (s.iter >= opt.max_num_iterations) return stop(LM_MAX_ITER, SFMB200_BA_NO_CONVERGENCE);
        }
    }
    if (s.gmax <= opt.gradient_tolerance) return stop(LM_GRADIENT_TOL, SFMB200_BA_CONVERGENCE);
    if (s.radius <= opt.min_trust_region_radius) return stop(LM_MIN_RADIUS, SFMB200_BA_CONVERGENCE);
    ++s.iter;
    const bool lin_ok = fail0 == 0.0 && fail1 == 0.0 && isfinite(model_acc) && isfinite(dn2_pts) && isfinite(dn2_cf);
    const double model_cost_change = -model_acc;
    bool decided = false;
    if (!lin_ok || !(model_cost_change > 0.0)) {
        s.num_unsuccessful++;
        if (++s.invalid_steps >= opt.max_num_consecutive_invalid_steps) return stop(LM_INVALID_STEPS, SFMB200_BA_FAILURE);
        s.radius /= s.decrease_factor; s.decrease_factor *= 2.0;
        decided = true;
    }
    if (!decided) {
        s.invalid_steps = 0;
        const double step_norm = sqrt(dn2_pts + dn2_cf);
        const double cand_cost = isfinite(cand_cost_raw) ? cand_cost_raw : 1.7976931348623157e308;
        if (step_norm <= opt.parameter_tolerance * (s.x_norm + opt.parameter_tolerance)) {
            s.msg_a = step_norm / (s.x_norm + opt.parameter_tolerance); s.msg_b = opt.parameter_tolerance;
            return stop(LM_PARAMETER_TOL, SFMB200_BA_CONVERGENCE);
        }
        const double cost_change = s.x_cost - cand_cost;
        if (fabs(cost_change) <= opt.function_tolerance * s.x_cost) {
            s.msg_a = fabs(cost_change) / s.x_cost; s.msg_b = opt.function_tolerance;
            return stop(LM_FUNCTION_TOL, SFMB200_BA_CONVERGENCE);
        }
        const double relative_decrease = cost_change / model_cost_change;
        s.last_rho = relative_decrease;
        if (relative_decrease > opt.min_relative_decrease) {
            s.cur ^= 1;                              // x <- candidate
            s.x_norm = sqrt(cn2_pts + cn2_cf); s.new_point = 1;
            const double q = 2.0 * relative_decrease - 1.0;
            s.radius = fmin(opt.max_trust_region_radius, s.radius / fmax(1.0 / 3.0, 1.0 - q * q * q));
            s.decrease_factor = 2.0;
            s.num_successful++;
            s.x_cost = cand_cost;                   // refreshed from the pass at the new point next iteration
        } else {
            s.radius /= s.decrease_factor; s.decrease_factor *= 2.0;
            s.num_unsuccessful++;
        }
    }
    // FinalizeIterationAndCheckIfMinimizerCanContinue of the next iteration (the time limit is the host's, between chunks)
    if (s.iter >= opt.max_num_iterations) return stop(LM_MAX_ITER, SFMB200_BA_NO_CONVERGENCE);
    *st = s;
}

// ---------------------------------------------------------------------------------------------------------------
// Back substitution for the points + step evaluation from STORED blocks (gather mode, default): no Jacobian is evaluated.
// With Z_o = Jc^T Jp M^T (Zbuf, written by K3a) and M, zg = M g, zf = M wf, g, diag(U) per point (ptblk):
//     y_p = M^T (zg - sum_o Z_o^T y_c(o) - zf y_f)                  [ M sum_o Jp^T (Jc y_c + Jf y_f) = sum_o Z_o^T y_c + zf y_f ]
// and, because y solves (J^T J + D^2) y = g exactly (direct solve), Ceres' model cost change  -m.(r + m/2), m = -J y,  equals
//     1/2 y.(g + D^2 y)        summed over all parameters, D^2 = clamp(diag(J^T J)) / radius
// -- the point part is accumulated here, the camera/focal part by ba_cam_update_kernel (locals[4]).  What remains per
// observation is one 144-byte record, 18 FMAs and the residual at the candidate: 93 -> ~50 us at cfg 3 (HBM: Zbuf 230 MB).
// post[0] = sum r'^2, post[1] = -(point part of the model cost change), post[2] = |delta_pts|^2, post[3] = |cand_pts|^2
// ---------------------------------------------------------------------------------------------------------------
// Per-camera operands (candidate rotation + translation, y_c: 18 doubles) are staged in shared memory once per CTA when they
// fit (CAMTAB): gathered per observation from global memory they were 12 of the 24 L1 sectors per observation of a kernel that
// is L1-throughput bound (ncu: l1tex 77 %).
template <int G, bool CAMTAB>
__global__ void __launch_bounds__(PT_THREADS) ba_backsub_z_kernel(BAView v, double inv_radius, const double* __restrict__ y_cf, const double* cand_cf,
                                                                  const CamDerived* camd_c, double* pts_c, double* __restrict__ post) {
    extern __shared__ __align__(16) double camtab[];                  // [nc][18]: R(9) t(3) y_c(6)   (CAMTAB)
    const LMX x = lm_x(v);
    if (!x.run) return;
    if (v.st) { const int nxt = v.st->cur ^ 1; cand_cf = v.cf2[nxt]; camd_c = v.camd2[nxt]; pts_c = v.pts2[nxt]; inv_radius = 1.0 / v.st->radius; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gl = lane % G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << ((lane / G) * G));
    constexpr int GB = PT_THREADS / G;
    const double yf = y_cf[6 * v.nc], fc = cand_cf[6 * v.nc];
    if (CAMTAB) {
        for (int i = threadIdx.x; i < v.nc * 18; i += PT_THREADS) {
            const int c = i / 18, q = i - 18 * c;
            camtab[i] = q < 12 ? reinterpret_cast<const double*>(camd_c + c)[q] : y_cf[6 * c + q - 12];
        }
        __syncthreads();
    }
    double acc_cc = 0, acc_m = 0, acc_dn = 0, acc_cn = 0;
    constexpr int GW = 32 / G;
    __shared__ __align__(16) double zstage[PT_THREADS / 32][32 * 18];
    const int np_round = (v.np + GB - 1) / GB * GB;
    // The iteration is a chain of dependent loads (offsets -> records / indices -> per-camera data); with 24 warps per SM that
    // latency is exposed, so the NEXT iteration's lines are pulled into L2 while this one computes (prefetch.global.L2: no
    // registers), and its CSR offsets are loaded one iteration ahead.
    int o0_next = 0, k_next = 0;
    { const int pn = blockIdx.x * GB + threadIdx.x / G; if (pn < v.np) { o0_next = v.pt_off[pn]; k_next = v.pt_off[pn + 1] - o0_next; } }
    for (int p0 = blockIdx.x * GB; p0 < np_round; p0 += gridDim.x * GB) {
        const int p = p0 + threadIdx.x / G;
        const bool active = p < v.np;
        const int o0 = o0_next, k = k_next;
        {
            const int pn = p + gridDim.x * GB;
            o0_next = 0; k_next = 0;
            if (pn < v.np) {
                o0_next = v.pt_off[pn]; k_next = v.pt_off[pn + 1] - o0_next;
                if (gl < k_next) {
                    const char* zr = reinterpret_cast<const char*>(v.Zbuf + (size_t)(o0_next + gl) * 18);
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(zr)); asm volatile("prefetch.global.L2 [%0];" :: "l"(zr + 128));
                }
                if (gl == 0) {
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(v.obs_cam + o0_next)); asm volatile("prefetch.global.L2 [%0];" :: "l"(v.obs_xy + o0_next));
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(x.pts + 3 * (size_t)pn)); asm volatile("prefetch.global.L2 [%0];" :: "l"(v.scale_pt + 3 * (size_t)pn));
                    const char* pbn = reinterpret_cast<const char*>(v.ptblk + (size_t)pn * PTB);
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(pbn)); asm volatile("prefetch.global.L2 [%0];" :: "l"(pbn + 128));
                }
            }
        }
        // the warp's Z records are one contiguous range (at most G observations per point): coalesced load into shared memory,
        // then every lane reads its own record (conflict free) -- a lane-per-record global load touches 36 lines per instruction
        const bool stage = v.maxk <= G;
        int o_first = 0;
        if (stage) {
            // the warp's range of records: from its first group's offset to the end of its last active group (no extra loads)
            o_first = __shfl_sync(0xffffffffu, o0, 0);
            const int o_end = (int)__reduce_max_sync(0xffffffffu, (unsigned)(o0 + k));
            __syncwarp();
            const double2* in = reinterpret_cast<const double2*>(v.Zbuf + (size_t)o_first * 18);
            double2* dstz = reinterpret_cast<double2*>(zstage[warp]);
            for (int i = lane; i < (o_end - o_first) * 9; i += 32) dstz[i] = in[i];
            __syncwarp();
        }
        double t[3] = {0, 0, 0};
        for (int j = gl; j < k; j += G) {
            const int o = o0 + j, c = v.obs_cam[o];
            const double2* z = stage ? reinterpret_cast<const double2*>(zstage[warp] + (size_t)(o - o_first) * 18)
                                     : reinterpret_cast<const double2*>(v.Zbuf + (size_t)o * 18);
#pragma unroll
            for (int a = 0; a < 6; a += 2) {          // rows a, a+1 = six doubles = three 16-byte loads
                const double2 z0 = z[a / 2 * 3], z1 = z[a / 2 * 3 + 1], z2 = z[a / 2 * 3 + 2];
                const double ya = CAMTAB ? camtab[18 * c + 12 + a] : y_cf[6 * c + a], yb = CAMTAB ? camtab[18 * c + 13 + a] : y_cf[6 * c + a + 1];
                t[0] += z0.x * ya + z1.y * yb; t[1] += z0.y * ya + z2.x * yb; t[2] += z1.x * ya + z2.y * yb;
            }
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) t[a] = group_sum<G>(t[a], gmask);
        if (!active) continue;
        const double X[3] = {x.pts[3 * p], x.pts[3 * p + 1], x.pts[3 * p + 2]};
        const double sp[3] = {v.scale_pt[3 * p], v.scale_pt[3 * p + 1], v.scale_pt[3 * p + 2]};
        const double* pb = v.ptblk + (size_t)p * PTB;
        const double M[6] = {pb[0], pb[1], pb[2], pb[3], pb[4], pb[5]};
        const double u0 = pb[6] - t[0] - pb[9] * yf, u1 = pb[7] - t[1] - pb[10] * yf, u2 = pb[8] - t[2] - pb[11] * yf;
        const double yp[3] = {M[0] * u0 + M[1] * u1 + M[3] * u2, M[2] * u1 + M[4] * u2, M[5] * u2};
        const double Xc[3] = {X[0] - yp[0] * sp[0], X[1] - yp[1] * sp[1], X[2] - yp[2] * sp[2]};
        if (gl == 0) {
            pts_c[3 * p] = Xc[0]; pts_c[3 * p + 1] = Xc[1]; pts_c[3 * p + 2] = Xc[2];
            const double d0 = X[0] - Xc[0], d1 = X[1] - Xc[1], d2 = X[2] - Xc[2];
            acc_dn += d0 * d0 + d1 * d1 + d2 * d2;
            acc_cn += Xc[0] * Xc[0] + Xc[1] * Xc[1] + Xc[2] * Xc[2];
#pragma unroll
            for (int a = 0; a < 3; ++a) acc_m -= 0.5 * yp[a] * (pb[12 + a] + clampd(pb[15 + a], v.min_diag, v.max_diag) * inv_radius * yp[a]);
        }
        for (int j = gl; j < k; j += G) {
            const int o = o0 + j, c = v.obs_cam[o];
            const float2 xy = v.obs_xy[o];
            double rc[2];
            if (CAMTAB) {
                const double* ct = camtab + 18 * c;                    // same arithmetic as obs_residual
                const double p0 = ct[0] * Xc[0] + ct[1] * Xc[1] + ct[2] * Xc[2] + ct[9];
                const double p1 = ct[3] * Xc[0] + ct[4] * Xc[1] + ct[5] * Xc[2] + ct[10];
                const double p2 = ct[6] * Xc[0] + ct[7] * Xc[1] + ct[8] * Xc[2] + ct[11];
                const double iz = 1.0 / p2;
                rc[0] = fc * (p0 * iz) - (double)xy.x; rc[1] = fc * (p1 * iz) - (double)xy.y;
            } else obs_residual(camd_c[c], Xc, fc, (double)xy.x, (double)xy.y, rc);
            acc_cc += rc[0] * rc[0] + rc[1] * rc[1];
        }
    }
    __shared__ double sred[PT_THREADS / 32][4];
    const double c0 = warp_sum(acc_cc), c1 = warp_sum(acc_m), c2 = warp_sum(acc_dn), c3 = warp_sum(acc_cn);
    if (lane == 0) { sred[warp][0] = c0; sred[warp][1] = c1; sred[warp][2] = c2; sred[warp][3] = c3; }
    __syncthreads();
    double t[4] = {0, 0, 0, 0};
    if (threadIdx.x == 0) for (int w = 0; w < PT_THREADS / 32; ++w) { t[0] += sred[w][0]; t[1] += sred[w][1]; t[2] += sred[w][2]; t[3] += sred[w][3]; }
    double tot[4];
    if (last_block_sum4(v.part4, v.counters + 1, t, tot) && threadIdx.x == 0) { post[0] = tot[0]; post[1] = tot[1]; post[2] = tot[2]; post[3] = tot[3]; }
}

// ---------------------------------------------------------------------------------------------------------------
// Back substitution for the points + step evaluation from re-evaluated Jacobians (default; no Z blocks are read):
//     y_p = M^T (zg - M t),   t = sum_o Jp^T (Jc y_c + Jf y_f)        [ M t = sum_o Z_o^T y_c + zf y_f ]
// One closed-form Jacobian at x per observation (~300 flop) instead of a 144-byte Z record, then the residual at the candidate.
// The model cost change is the same 1/2 y.(g + D^2 y) as in ba_backsub_z_kernel (point part here, camera/focal part in
// ba_cam_update_kernel), so the Jacobian is not needed a second time.
// Per-camera operands (CamDerived at x, candidate rotation + translation, scaled y_c) sit in shared memory when they fit
// (CAMTAB); the next iteration's lines are prefetched into L2 and its CSR offsets loaded one iteration ahead, as in
// ba_backsub_z_kernel.
// post[0] = sum r'^2, post[1] = -(point part of the model cost change), post[2] = |delta_pts|^2, post[3] = |cand_pts|^2
// ---------------------------------------------------------------------------------------------------------------
struct BacksubCam {
    CamDerived d;                  // at x
    double Rc[9], tc[3];           // candidate rotation and translation
    double ys[6];                  // scale_cf * y_c
};
template <int G, bool CAMTAB>
__global__ void __launch_bounds__(PT_THREADS) ba_backsub_eval_kernel(BAView v, double inv_radius, const double* __restrict__ y_cf, const double* cand_cf,
                                                                     const CamDerived* camd_c, double* pts_c, double* __restrict__ post) {
    extern __shared__ __align__(16) unsigned char bs_smem[];
    BacksubCam* camtab = reinterpret_cast<BacksubCam*>(bs_smem);     // [nc] (CAMTAB)
    const LMX x = lm_x(v);
    if (!x.run) return;
    if (v.st) { const int nxt = v.st->cur ^ 1; cand_cf = v.cf2[nxt]; camd_c = v.camd2[nxt]; pts_c = v.pts2[nxt]; inv_radius = 1.0 / v.st->radius; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gl = lane % G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << ((lane / G) * G));
    constexpr int GB = PT_THREADS / G;
    const double f = *x.focal, yfs = v.scale_cf[6 * v.nc] * y_cf[6 * v.nc], fc = cand_cf[6 * v.nc];
    if (CAMTAB) {
        constexpr int CD = sizeof(CamDerived) / 8, CT = sizeof(BacksubCam) / 8;
        double* tab = reinterpret_cast<double*>(bs_smem);
        for (int i = threadIdx.x; i < v.nc * CT; i += PT_THREADS) {
            const int c = i / CT, q = i - CT * c;
            tab[i] = q < CD ? reinterpret_cast<const double*>(x.camd + c)[q]
                   : q < CD + 12 ? reinterpret_cast<const double*>(camd_c + c)[q - CD]
                   : v.scale_cf[6 * c + q - CD - 12] * y_cf[6 * c + q - CD - 12];
        }
        __syncthreads();
    }
    double acc_cc = 0, acc_m = 0, acc_dn = 0, acc_cn = 0;
    const int np_round = (v.np + GB - 1) / GB * GB;
    int o0_next = 0, k_next = 0;
    { const int pn = blockIdx.x * GB + threadIdx.x / G; if (pn < v.np) { o0_next = v.pt_off[pn]; k_next = v.pt_off[pn + 1] - o0_next; } }
    for (int p0 = blockIdx.x * GB; p0 < np_round; p0 += gridDim.x * GB) {
        const int p = p0 + threadIdx.x / G;
        const bool active = p < v.np;
        const int o0 = o0_next, k = k_next;
        {
            const int pn = p + gridDim.x * GB;
            o0_next = 0; k_next = 0;
            if (pn < v.np) {
                o0_next = v.pt_off[pn]; k_next = v.pt_off[pn + 1] - o0_next;
                if (gl == 0) {
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(v.obs_cam + o0_next)); asm volatile("prefetch.global.L2 [%0];" :: "l"(v.obs_xy + o0_next));
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(x.pts + 3 * (size_t)pn)); asm volatile("prefetch.global.L2 [%0];" :: "l"(v.scale_pt + 3 * (size_t)pn));
                    const char* pbn = reinterpret_cast<const char*>(v.ptblk + (size_t)pn * PTB);
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(pbn)); asm volatile("prefetch.global.L2 [%0];" :: "l"(pbn + 128));
                }
            }
        }
        double X[3] = {0, 0, 0};
        if (active) { X[0] = x.pts[3 * p]; X[1] = x.pts[3 * p + 1]; X[2] = x.pts[3 * p + 2]; }
        // pass 1: t = sum_o Jp^T (Jc y_c + Jf y_f), Jacobians unscaled; the scaling is folded into ys, yfs and sp
        double t[3] = {0, 0, 0};
        for (int j = gl; j < k; j += G) {
            const int o = o0 + j, c = v.obs_cam[o];
            const float2 xy = v.obs_xy[o];
            double r[2], Jc[12], Jp[6], Jf[2];
            obs_eval(CAMTAB ? camtab[c].d : x.camd[c], X, f, (double)xy.x, (double)xy.y, r, Jc, Jp, Jf);
            double m0 = Jf[0] * yfs, m1 = Jf[1] * yfs;
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                const double ys = CAMTAB ? camtab[c].ys[a] : v.scale_cf[6 * c + a] * y_cf[6 * c + a];
                m0 += Jc[a] * ys; m1 += Jc[6 + a] * ys;
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) t[a] += Jp[a] * m0 + Jp[3 + a] * m1;
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) t[a] = group_sum<G>(t[a], gmask);
        if (!active) continue;
        const double sp[3] = {v.scale_pt[3 * p], v.scale_pt[3 * p + 1], v.scale_pt[3 * p + 2]};
        t[0] *= sp[0]; t[1] *= sp[1]; t[2] *= sp[2];
        const double* pb = v.ptblk + (size_t)p * PTB;
        const double M[6] = {pb[0], pb[1], pb[2], pb[3], pb[4], pb[5]};
        // u = zg - M t ; y_p = M^T u
        const double u0 = pb[6] - M[0] * t[0], u1 = pb[7] - (M[1] * t[0] + M[2] * t[1]), u2 = pb[8] - (M[3] * t[0] + M[4] * t[1] + M[5] * t[2]);
        const double yp[3] = {M[0] * u0 + M[1] * u1 + M[3] * u2, M[2] * u1 + M[4] * u2, M[5] * u2};
        const double Xc[3] = {X[0] - yp[0] * sp[0], X[1] - yp[1] * sp[1], X[2] - yp[2] * sp[2]};
        if (gl == 0) {
            pts_c[3 * p] = Xc[0]; pts_c[3 * p + 1] = Xc[1]; pts_c[3 * p + 2] = Xc[2];
            const double d0 = X[0] - Xc[0], d1 = X[1] - Xc[1], d2 = X[2] - Xc[2];
            acc_dn += d0 * d0 + d1 * d1 + d2 * d2;
            acc_cn += Xc[0] * Xc[0] + Xc[1] * Xc[1] + Xc[2] * Xc[2];
#pragma unroll
            for (int a = 0; a < 3; ++a) acc_m -= 0.5 * yp[a] * (pb[12 + a] + clampd(pb[15 + a], v.min_diag, v.max_diag) * inv_radius * yp[a]);
        }
        // pass 2: residual at the candidate
        for (int j = gl; j < k; j += G) {
            const int o = o0 + j, c = v.obs_cam[o];
            const float2 xy = v.obs_xy[o];
            double rc[2];
            if (CAMTAB) {
                const double* Rc = camtab[c].Rc; const double* tc = camtab[c].tc;       // same arithmetic as obs_residual
                const double q0 = Rc[0] * Xc[0] + Rc[1] * Xc[1] + Rc[2] * Xc[2] + tc[0];
                const double q1 = Rc[3] * Xc[0] + Rc[4] * Xc[1] + Rc[5] * Xc[2] + tc[1];
                const double q2 = Rc[6] * Xc[0] + Rc[7] * Xc[1] + Rc[8] * Xc[2] + tc[2];
                const double iz = 1.0 / q2;
                rc[0] = fc * (q0 * iz) - (double)xy.x; rc[1] = fc * (q1 * iz) - (double)xy.y;
            } else obs_residual(camd_c[c], Xc, fc, (double)xy.x, (double)xy.y, rc);
            acc_cc += rc[0] * rc[0] + rc[1] * rc[1];
        }
    }
    __shared__ double sred[PT_THREADS / 32][4];
    const double c0 = warp_sum(acc_cc), c1 = warp_sum(acc_m), c2 = warp_sum(acc_dn), c3 = warp_sum(acc_cn);
    if (lane == 0) { sred[warp][0] = c0; sred[warp][1] = c1; sred[warp][2] = c2; sred[warp][3] = c3; }
    __syncthreads();
    double tt[4] = {0, 0, 0, 0};
    if (threadIdx.x == 0) for (int w = 0; w < PT_THREADS / 32; ++w) { tt[0] += sred[w][0]; tt[1] += sred[w][1]; tt[2] += sred[w][2]; tt[3] += sred[w][3]; }
    double tot[4];
    if (last_block_sum4(v.part4, v.counters + 1, tt, tot) && threadIdx.x == 0) { post[0] = tot[0]; post[1] = tot[1]; post[2] = tot[2]; post[3] = tot[3]; }
}

// camera-major copy of the observation list: counting sort by camera (structure is fixed across LM iterations).
// Shared-memory histograms per CTA keep the same-address global atomics down to (CTAs x cameras) instead of one per
// observation (1.6M atomics on 100 counters took 300 us each way).
constexpr int SORT_THREADS = 1024;
__global__ void __launch_bounds__(SORT_THREADS) count_cams_kernel(const int32_t* __restrict__ obs_cam, int nobs, int nc, int use_smem, int* __restrict__ cnt) {
    extern __shared__ int sh[];
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (!use_smem) { if (o < nobs) atomicAdd(cnt + obs_cam[o], 1); return; }
    for (int i = threadIdx.x; i < nc; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    if (o < nobs) atomicAdd(sh + obs_cam[o], 1);
    __syncthreads();
    for (int i = threadIdx.x; i < nc; i += blockDim.x) if (sh[i]) atomicAdd(cnt + i, sh[i]);
}
__global__ void scan_small_kernel(const int* __restrict__ cnt, int n, int32_t* __restrict__ off, int* __restrict__ cursor) {
    if (threadIdx.x == 0 && blockIdx.x == 0) { int s = 0; for (int i = 0; i < n; ++i) { off[i] = s; cursor[i] = s; s += cnt[i]; } off[n] = s; }
}
__global__ void expand_obs_pt_kernel(const int32_t* __restrict__ pt_off, int np, int32_t* __restrict__ obs_pt) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < np) for (int o = pt_off[p]; o < pt_off[p + 1]; ++o) obs_pt[o] = p;
}
__global__ void __launch_bounds__(SORT_THREADS) scatter_cm_kernel(const int32_t* __restrict__ obs_cam, const float2* __restrict__ obs_xy,
                                                                  const int32_t* __restrict__ obs_pt, int nobs, int nc, int use_smem,
                                                                  int* __restrict__ cursor, float2* __restrict__ cm_xy, int32_t* __restrict__ cm_pt) {
    extern __shared__ int sh[];          // [2*nc]: per-CTA count, then reserved base
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (!use_smem) {
        if (o < nobs) { const int pos = atomicAdd(cursor + obs_cam[o], 1); cm_xy[pos] = obs_xy[o]; cm_pt[pos] = obs_pt[o]; }
        return;
    }
    for (int i = threadIdx.x; i < nc; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    int c = 0, r = 0;
    if (o < nobs) { c = obs_cam[o]; r = atomicAdd(sh + c, 1); }
    __syncthreads();
    for (int i = threadIdx.x; i < nc; i += blockDim.x) if (sh[i]) sh[nc + i] = atomicAdd(cursor + i, sh[i]);
    __syncthreads();
    if (o < nobs) { const int pos = sh[nc + c] + r; cm_xy[pos] = obs_xy[o]; cm_pt[pos] = obs_pt[o]; }
}

// ---------------------------------------------------------------------------------------------------------------
// Cross-GPU sum over PEER MEMORY (one process per GPU, buffers mapped with CUDA IPC, loads travel over NVLink/NVSwitch).
// Replaces ncclAllReduce for the reduced camera system: every rank reads the partial buffers of all ranks directly and
// sums them in the same order (bitwise identical result on every rank), ~2 us of flag traffic instead of a collective
// launch.  Protocol per call (epoch e, monotonically increasing, same sequence on every rank):
//   peer_signal(A,e)  "my partial buffer is complete"      -> written into every peer's flag array
//   peer_reduce       waits A>=e from all ranks, tmp[i] = sum_r buf_r[i]  (max for the tail range)
//   peer_signal(B,e)  "I have finished reading everybody's buffer"
//   peer_copyback     waits B>=e from all ranks, buf <- tmp   (nobody reads my partials any more)
// ---------------------------------------------------------------------------------------------------------------
constexpr int MAX_PEERS = 16;
struct PeerTable { double* buf[MAX_PEERS]; unsigned long long* flags[MAX_PEERS]; };   // flags: [2][MAX_PEERS] per rank

__device__ __forceinline__ unsigned long long ld_flag(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// The reduction kernel first tells the peers that THIS rank's partial buffer is final (stream order guarantees it), then waits
// until every rank has said the same, then sums the peers' buffers in rank order into a rank-LOCAL copy (P->xtmp, same
// offsets as the exchange buffer) that the consumers read -- nothing is written back into the exchanged buffer, so no second
// "done reading" handshake is needed: a rank overwrites a region of its exchange buffer only after a LATER hand-shake in
// which every peer took part after finishing its reads (red: cleared after the post reduction of the same iteration; post:
// cleared by ba_cam_update_kernel after the red reduction of the next one).  One launch and one hand-shake per all-reduce.
__device__ __forceinline__ void peer_signal(const PeerTable& t, int slot, int my_rank, int nranks, unsigned long long epoch) {
    if (blockIdx.x == 0 && (int)threadIdx.x < nranks) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(t.flags[threadIdx.x] + slot * MAX_PEERS + my_rank), "l"(epoch) : "memory");
    }
}
// Bounded: a peer that never arrives (a rank died) must not hang the GPU -- after ~20 s the wait gives up and raises the
// dense-solve failure counter, which makes the LM loop reject the step and terminate with FAILURE.
__device__ __forceinline__ void peer_wait(const unsigned long long* my_flags, int slot, int nranks, unsigned long long epoch, int* fail) {
    if ((int)threadIdx.x < nranks) {
        const long long t0 = clock64();
        while (ld_flag(my_flags + slot * MAX_PEERS + threadIdx.x) < epoch) {
            __nanosleep(64);
            if (clock64() - t0 > 40000000000LL) { if (fail && blockIdx.x == 0) atomicAdd(fail, 1000); break; }
        }
    }
    __syncthreads();
    __threadfence_system();
}
__global__ void __launch_bounds__(256) peer_reduce_kernel(PeerTable t, size_t offset, int my_rank, int nranks, unsigned long long epoch,
                                                          size_t n_sum, size_t n_max, double* __restrict__ out, int* __restrict__ fail) {
    peer_signal(t, 0, my_rank, nranks, epoch);
    peer_wait(t.flags[my_rank], 0, nranks, epoch, fail);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sum + n_max; i += (size_t)gridDim.x * blockDim.x) {
        double acc = __ldcv(t.buf[0] + offset + i);
        for (int r = 1; r < nranks; ++r) { const double v = __ldcv(t.buf[r] + offset + i); acc = i < n_sum ? acc + v : fmax(acc, v); }
        out[i] = acc;
    }
}

}  // namespace

// =================================================================================================================
// events of one LM iteration: 0 point start, 1 point end, 2 pair end, 3 camera end, 4 solve start, 5 solve end, 6/7 flush
constexpr int LM_CHUNK = 4;            // LM iterations enqueued per host read-back (large problems)
constexpr int LM_CHUNK_MAX = 16;       // small problems (adjustBundle inside runSfM: a few thousand observations, ~100 iterations): their
                                       // iteration is a chain of launch-bound kernels, the read-back + sync per chunk is a visible share
struct EvSet { cudaEvent_t ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}; };

struct sfmb200_ba_problem {
    sfmb200_ctx* ctx = nullptr;
    int nc = 0, np = 0, nobs = 0, maxk = 0, G = 8, n = 0, npad = 0;
    DevBuf mem;                       // one allocation, carved below
    DevBuf xbuf; PinBuf hpin; bool borrowed = false;   // exchange memory / pinned read-back; workspace borrowed from ctx->ba_ws
    // observations
    float2* obs_xy; int32_t* obs_cam; int32_t* pt_off; int32_t* cm_off; float2* cm_xy; int32_t* cm_pt;
    // state: x = (cf, pts), candidate, initial
    double* cf[2]; double* pts[2]; double* cf0; double* pts0; int cur = 0; double focal0 = 0;
    CamDerived* camd[2];
    double* scale_cf; double* scale_pt; double* ptblk;
    // reduced system buffer (one all-reduce): Sblk | Scf | Sff | rhs | gcf | dcf | sums[8]
    double* red; size_t red_n; double* Sblk; double* Scf; double* Sff; double* rhs; double* gcf; double* dcf; double* sums;
    double* post;                     // [8] summed over ranks
    double* locals;                   // [8] identical on every rank
    unsigned long long* gmax_pt_bits; int* fail;   // fail[0] point blocks, fail[1] dense Cholesky
    double* A; double* y_cf; double* dinv;
    int grid_point = 0, grid_backsub = 0, grid_camera = 0;   // persistent grids = co-resident CTA count
    double* Linv = nullptr;           // [npad/NB][NB][NB] inverses of the diagonal tiles (dataflow Cholesky -> back substitution)
    bool backsolve_cluster = false;   // back substitution on a CTA cluster (small enough n) or on one CTA
    uint4* chol_ll = nullptr; int chol_grid_stream = 0;
    unsigned* chol_ready = nullptr; unsigned chol_epoch = 0;   // dataflow Cholesky (K4)
    unsigned* solve_counter = nullptr;   // device-side number of the current dense solve (incremented by ba_assemble_kernel)
    double* h_scal = nullptr;         // pinned read-back: sums[8] post[8] locals[8] gmax fail
    bool have_scale = false;
    bool backsub_from_z = false;      // back-substitution from the stored Z blocks (gather mode, Zbuf within one L2-sized segment) instead of re-evaluated Jacobians
    bool camd_valid[2] = {false, false};   // camd[i] matches cf[i] (written by cam_derive or, for the candidate, by ba_cam_update_kernel)
    EvSet evs[LM_CHUNK_MAX];              // profile mode: one set of events per iteration of a chunk (created on first use)
    bool have_events = false;
    LMState* d_state = nullptr; LMState* h_state = nullptr;    // device-resident LM control state + pinned read-back
    // row mode (default): Z per observation (point-major), stable camera-major list with follower counts, partial records
    bool gather = true;               // true = gather mode (ba_pair_kernel + partial records), false = "red" mode
    double* Zbuf = nullptr;
    int32_t* obs_pt = nullptr; int32_t* cm_obs = nullptr; uint8_t* cm_np = nullptr;
    double* diag_part = nullptr; int diag_grid = 0, diag_per_cta = 0;
    int32_t* pair_off = nullptr; int32_t* pair_blk = nullptr; uint2* pair_ent = nullptr; double* pair_part = nullptr;
    int n_pairs_nonempty = 0, pair_splits = 1, pair_nseg = 1;
    double* part4 = nullptr; double* fpart = nullptr; unsigned* counters = nullptr;
    DevBuf gmem;
    // exchange memory (its own cudaMalloc so that it can be exported with CUDA IPC): red | post.. | flags
    void* xmem = nullptr; size_t xmem_doubles = 0; double* xtmp = nullptr; unsigned long long* xflags = nullptr;
    bool peers = false; PeerTable ptab; void* peer_base[MAX_PEERS] = {nullptr}; unsigned long long epoch = 0;
};

// give the buffers back to the context's cache (or free them when this problem allocated its own)
static void ba_release_buffers(sfmb200_ba_problem* P) {
    sfmb200_ctx* ctx = P->ctx;
    if (P->borrowed) {
        ctx->ba_ws.mem = P->mem; ctx->ba_ws.gmem = P->gmem; ctx->ba_ws.xbuf = P->xbuf; ctx->ba_ws.hpin = P->hpin;
        ctx->ba_ws.in_use = false;
    } else { P->mem.release(); P->gmem.release(); P->xbuf.release(); P->hpin.release(); }
    P->mem = DevBuf(); P->gmem = DevBuf(); P->xbuf = DevBuf(); P->hpin = PinBuf(); P->xmem = nullptr; P->h_scal = nullptr; P->borrowed = false;
}

static BAView make_view(const sfmb200_ba_problem* P, const sfmb200_ba_options* opt, bool lm = false) {
    BAView v;
    v.st = lm ? P->d_state : nullptr;
    for (int i = 0; i < 2; ++i) { v.cf2[i] = P->cf[i]; v.pts2[i] = P->pts[i]; v.camd2[i] = P->camd[i]; }
    v.nc = P->nc; v.np = P->np; v.nobs = P->nobs; v.maxk = P->maxk;
    v.obs_xy = P->obs_xy; v.obs_cam = P->obs_cam; v.pt_off = P->pt_off; v.cm_off = P->cm_off; v.cm_xy = P->cm_xy; v.cm_pt = P->cm_pt;
    v.cams = P->cf[P->cur]; v.focal = P->cf[P->cur] + 6 * P->nc; v.pts = P->pts[P->cur]; v.camd = P->camd[P->cur];
    v.scale_cf = P->scale_cf; v.scale_pt = P->scale_pt; v.ptblk = P->ptblk; v.Zbuf = P->Zbuf;
    v.Sblk = P->Sblk; v.Scf = P->Scf; v.Sff = P->Sff; v.rhs = P->rhs; v.gcf = P->gcf; v.dcf = P->dcf; v.sums = P->sums;
    v.gmax_pt_bits = P->gmax_pt_bits; v.fail = P->fail;
    v.min_diag = opt->min_lm_diagonal; v.max_diag = opt->max_lm_diagonal;
    v.part4 = P->part4; v.counters = P->counters;
    return v;
}

static RowArgs make_row_args(const sfmb200_ba_problem* P) {
    RowArgs ra; ra.diag_per_cta = P->diag_per_cta; ra.diag_part = P->diag_part;
    ra.pair_off = P->pair_off; ra.pair_part = P->pair_part; ra.nseg = P->pair_nseg; ra.splits = P->pair_splits;
    ra.pair_blk = P->pair_blk; ra.n_nonempty = P->n_pairs_nonempty;
    return ra;
}

// Point segments of the pair accumulation: Zbuf (144 bytes per observation) in slices of a quarter of the L2 cache, so that the
// slice all resident warps of ba_pair_kernel read stays L2-resident next to the streamed entry lists (H100: 50 MB L2 in two
// partitions -> 12.5 MB slices).
static int pair_segments(const sfmb200_ctx* ctx, int nobs) {
    const long long seg = std::max(ctx->l2_bytes, 8 << 20) / 4;
    return (int)std::max<long long>(1, std::min<long long>(64, (144LL * nobs + seg - 1) / seg));
}

static size_t point_smem_bytes(int G, int maxk) {
    const int GB = PT_THREADS / G;
    return (size_t)GB * maxk * 18 * 8 + (size_t)GB * maxk * 4 + (size_t)maxk * (maxk - 1) / 2 * 2 + 16;
}

// Grid for a grid-stride kernel: exactly the number of co-resident CTAs (one balanced wave), cached per problem.
template <typename K> static int resident_grid(sfmb200_ba_problem* P, int* cache, K kernel, int threads, size_t smem, int work_blocks) {
    if (*cache == 0) {
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) { cudaGetLastError(); per_sm = 1; }
        *cache = per_sm * P->ctx->sm_count;
    }
    return std::max(1, std::min(work_blocks, *cache));
}

template <int G> static int launch_point_pass(sfmb200_ba_problem* P, const BAView& v, double inv_radius) {
    sfmb200_ctx* ctx = P->ctx;
    const int GB = PT_THREADS / G;
    if (P->gather) {
        const int blocks = resident_grid(P, &P->grid_point, ba_point_kernel<G, true>, PT_THREADS, 0, ceil_div(P->np, GB));
        ba_point_kernel<G, true><<<blocks, PT_THREADS, 0, ctx->stream>>>(v, inv_radius);
        SFM_LAUNCH_CHECK(ctx);
        return SFMB200_OK;
    }
    const size_t smem = point_smem_bytes(G, P->maxk);
    if (smem > 48 * 1024) SFM_CUDA(ctx, cudaFuncSetAttribute(ba_point_kernel<G, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int blocks = std::max(1, std::min(ceil_div(P->np, GB), ctx->sm_count * 8));
    ba_point_kernel<G, false><<<blocks, PT_THREADS, smem, ctx->stream>>>(v, inv_radius);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}
template <int G> static int launch_point_norm(sfmb200_ba_problem* P, const BAView& v) {
    sfmb200_ctx* ctx = P->ctx;
    const int GB = PT_THREADS / G;
    const int blocks = std::max(1, std::min(ceil_div(P->np, GB), ctx->sm_count * 16));
    ba_point_norm_kernel<G><<<blocks, PT_THREADS, 0, ctx->stream>>>(v, P->scale_pt);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}
template <int G> static int launch_backsub(sfmb200_ba_problem* P, const BAView& v) {
    sfmb200_ctx* ctx = P->ctx;
    const int GB = PT_THREADS / G, nxt = P->cur ^ 1;
    if (P->backsub_from_z) {            // gather mode: Z_o is in Zbuf, no Jacobian needed (inside the LM loop the radius comes from LMState)
        const size_t tab = sizeof(double) * 18 * (size_t)P->nc;
        if (tab <= 40 * 1024) {
            const int blocks = resident_grid(P, &P->grid_backsub, ba_backsub_z_kernel<G, true>, PT_THREADS, tab, ceil_div(P->np, GB));
            ba_backsub_z_kernel<G, true><<<blocks, PT_THREADS, tab, ctx->stream>>>(v, 0.0, P->y_cf, P->cf[nxt], P->camd[nxt], P->pts[nxt], P->post);
        } else {
            const int blocks = resident_grid(P, &P->grid_backsub, ba_backsub_z_kernel<G, false>, PT_THREADS, 0, ceil_div(P->np, GB));
            ba_backsub_z_kernel<G, false><<<blocks, PT_THREADS, 0, ctx->stream>>>(v, 0.0, P->y_cf, P->cf[nxt], P->camd[nxt], P->pts[nxt], P->post);
        }
    } else {                            // default: Jacobians re-evaluated at x (no Z blocks)
        const size_t tab = sizeof(BacksubCam) * (size_t)P->nc;
        if (tab <= 40 * 1024) {
            const int blocks = resident_grid(P, &P->grid_backsub, ba_backsub_eval_kernel<G, true>, PT_THREADS, tab, ceil_div(P->np, GB));
            ba_backsub_eval_kernel<G, true><<<blocks, PT_THREADS, tab, ctx->stream>>>(v, 0.0, P->y_cf, P->cf[nxt], P->camd[nxt], P->pts[nxt], P->post);
        } else {
            const int blocks = resident_grid(P, &P->grid_backsub, ba_backsub_eval_kernel<G, false>, PT_THREADS, 0, ceil_div(P->np, GB));
            ba_backsub_eval_kernel<G, false><<<blocks, PT_THREADS, 0, ctx->stream>>>(v, 0.0, P->y_cf, P->cf[nxt], P->camd[nxt], P->pts[nxt], P->post);
        }
    }
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}
#define DISPATCH_G(P, call)                                   \
    ((P)->G == 4 ? call<4> : (P)->G == 8 ? call<8> : (P)->G == 16 ? call<16> : call<32>)

static dim3 camera_grid(const sfmb200_ba_problem* P) {
    // enough CTAs per camera to fill the machine ~4x, at least one
    const int avg = P->nc > 0 ? std::max(1, P->nobs / std::max(1, P->nc)) : 1;
    int chunks = std::max(1, std::min(ceil_div(avg, CAM_THREADS), ceil_div(4 * P->ctx->sm_count, std::max(1, P->nc))));
    return dim3(chunks, std::max(1, P->nc));
}

// In-place reduction over ranks of buf[0..n_sum) (sum) and buf[n_sum..n_sum+n_max) (max); buf lives in the exchange memory.
static int ba_allreduce(sfmb200_ba_problem* P, double* buf, size_t n_sum, size_t n_max) {
    sfmb200_ctx* ctx = P->ctx;
    if (ctx->nranks <= 1) return SFMB200_OK;
    if (!P->peers) {                     // NCCL fallback
        int rc = sfmb200_allreduce_sum_f64(ctx, buf, n_sum); if (rc) return rc;
        return n_max ? sfmb200_allreduce_max_f64(ctx, buf + n_sum, n_max) : SFMB200_OK;
    }
    const size_t offset = buf - (double*)P->xmem, n = n_sum + n_max;
    const unsigned long long e = ++P->epoch;
    const int blocks = (int)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 4));
    peer_reduce_kernel<<<blocks, 256, 0, ctx->stream>>>(P->ptab, offset, ctx->rank, ctx->nranks, e, n_sum, n_max, P->xtmp + offset, P->fail + 1); SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

// Hand-shake only (peer exchange): after it every rank has finished the reads of all earlier reductions.  Needed where a region
// of the exchange buffer is overwritten without a later reduction in between (after the scaling pass; at the end of the
// reduced-system API call).
static int ba_peer_barrier(sfmb200_ba_problem* P) {
    sfmb200_ctx* ctx = P->ctx;
    if (ctx->nranks <= 1 || !P->peers) return SFMB200_OK;
    peer_reduce_kernel<<<1, 256, 0, ctx->stream>>>(P->ptab, 0, ctx->rank, ctx->nranks, ++P->epoch, 0, 0, P->xtmp, P->fail + 1); SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

// Where the rank-summed value of a location of the exchange buffer lives: in place (single GPU, NCCL) or in the local copy the
// peer reduction writes (same offset).
template <typename T> static T* summed(const sfmb200_ba_problem* P, T* p) {
    return P->peers ? reinterpret_cast<T*>(P->xtmp + (reinterpret_cast<double*>(p) - P->red)) : p;
}

// Jacobi scaling at the current x (iteration 0).  Multi-GPU: camera/focal column norms are summed over ranks.
static int compute_scaling(sfmb200_ba_problem* P, const sfmb200_ba_options* opt) {
    sfmb200_ctx* ctx = P->ctx;
    const int n = P->n;
    if (!opt->jacobi_scaling) {
        fill_kernel<<<ceil_div(n, 256), 256, 0, ctx->stream>>>(P->scale_cf, n, 1.0); SFM_LAUNCH_CHECK(ctx);
        if (P->np) { fill_kernel<<<ceil_div(3 * P->np, 256), 256, 0, ctx->stream>>>(P->scale_pt, 3 * (size_t)P->np, 1.0); SFM_LAUNCH_CHECK(ctx); }
        P->have_scale = true;
        return SFMB200_OK;
    }
    BAView v = make_view(P, opt);
    cam_derive_kernel<<<ceil_div(std::max(1, P->nc), 128), 128, 0, ctx->stream>>>(v.cams, P->nc, P->camd[P->cur]); SFM_LAUNCH_CHECK(ctx);
    P->camd_valid[P->cur] = true;
    double* colnorm = P->gcf;    // scratch: reuse (zeroed here, re-zeroed before every pass)
    SFM_CUDA(ctx, cudaMemsetAsync(colnorm, 0, sizeof(double) * n, ctx->stream));
    if (P->np > 0 && P->nobs > 0) {
        int rc = DISPATCH_G(P, launch_point_norm)(P, v); if (rc) return rc;
        if (P->gather) {                 // deterministic: partial records per (slice, camera), summed in slice order
            const RowArgs ra = make_row_args(P);
            ba_camera_kernel<true, true><<<P->diag_grid, CAM_THREADS, 0, ctx->stream>>>(v, P->diag_per_cta, P->diag_part); SFM_LAUNCH_CHECK(ctx);
            ba_combine_kernel<<<P->nc, COMBINE_THREADS, 0, ctx->stream>>>(v, ra, 1, colnorm, P->fpart, P->counters + 2); SFM_LAUNCH_CHECK(ctx);
        } else {
            ba_camera_norm_kernel<<<camera_grid(P), CAM_THREADS, 0, ctx->stream>>>(v, colnorm); SFM_LAUNCH_CHECK(ctx);
        }
    }
    int rc = ba_allreduce(P, colnorm, n, 0); if (rc) return rc;
    scale_from_norm_kernel<<<ceil_div(n, 256), 256, 0, ctx->stream>>>(summed(P, colnorm), n, P->scale_cf); SFM_LAUNCH_CHECK(ctx);
    P->have_scale = true;
    return ba_peer_barrier(P);          // the column norms sit in the region the first pass clears
}

// One residual+Jacobian+Schur pass at the current x; leaves the (rank-summed) reduced system in red.
// lm = true: inside the device-resident LM loop (x, radius and the early-out come from P->d_state, `radius` is ignored);
// es: CUDA events of this iteration's slot (profile mode) or nullptr.
static int schur_pass(sfmb200_ba_problem* P, const sfmb200_ba_options* opt, double radius, const EvSet* es, bool lm) {
    sfmb200_ctx* ctx = P->ctx;
    BAView v = make_view(P, opt, lm);
    const bool row = P->gather && P->np > 0 && P->nobs > 0;
    // "red" mode accumulates into the reduced system with atomics: clear all of it.  Row mode overwrites every element
    // (ba_combine_kernel), only locals | gmax | fail need clearing.  post is cleared by ba_cam_update_kernel.
    if (row) SFM_CUDA(ctx, cudaMemsetAsync(P->locals, 0, sizeof(double) * 12, ctx->stream));
    else SFM_CUDA(ctx, cudaMemsetAsync(P->red, 0, sizeof(double) * (P->red_n + 12), ctx->stream));
    if (!lm && !P->camd_valid[P->cur]) {
        cam_derive_kernel<<<ceil_div(std::max(1, P->nc), 128), 128, 0, ctx->stream>>>(v.cams, P->nc, P->camd[P->cur]); SFM_LAUNCH_CHECK(ctx);
        P->camd_valid[P->cur] = true;
    }
    if (P->np > 0 && P->nobs > 0) {
        if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[0], ctx->stream));
        int rc = DISPATCH_G(P, launch_point_pass)(P, v, 1.0 / radius); if (rc) return rc;
        if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[1], ctx->stream));
        if (row) {
            const RowArgs ra = make_row_args(P);
            if (P->n_pairs_nonempty > 0) {
                ba_pair_kernel<<<dim3(ceil_div(P->n_pairs_nonempty, PAIR_WARPS), P->pair_nseg * P->pair_splits), PAIR_WARPS * 32, 0, ctx->stream>>>(
                    P->Zbuf, P->pair_off, P->pair_ent, P->n_pairs_nonempty, P->pair_nseg, P->pair_splits, P->pair_blk, P->pair_part, v.st);
                SFM_LAUNCH_CHECK(ctx);
            }
            if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[2], ctx->stream));
            ba_camera_kernel<true, false><<<P->diag_grid, CAM_THREADS, 0, ctx->stream>>>(v, P->diag_per_cta, P->diag_part); SFM_LAUNCH_CHECK(ctx);
            ba_combine_kernel<<<P->nc + ceil_div(P->n_pairs_nonempty, COMBINE_THREADS / 32), COMBINE_THREADS, 0, ctx->stream>>>(v, ra, 0, nullptr, P->fpart, P->counters + 2); SFM_LAUNCH_CHECK(ctx);
        } else {
            if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[2], ctx->stream));
            const int blocks = resident_grid(P, &P->grid_camera, ba_camera_kernel<false, false>, CAM_THREADS, 0, ceil_div(P->nobs, CAM_THREADS));
            ba_camera_kernel<false, false><<<blocks, CAM_THREADS, 0, ctx->stream>>>(v, ceil_div(P->nobs, blocks), nullptr); SFM_LAUNCH_CHECK(ctx);
        }
        if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[3], ctx->stream));
    }
    return ba_allreduce(P, P->red, P->red_n, 0);
}

static int dense_solve(sfmb200_ba_problem* P, const sfmb200_ba_options* opt, double radius, bool lm) {
    sfmb200_ctx* ctx = P->ctx;
    const int npad = P->npad, nbk = npad / NB;
    const LMState* st = lm ? P->d_state : nullptr;
    const int* skip = lm ? &P->d_state->status : nullptr;
    ba_assemble_kernel<<<dim3(ceil_div(npad, 128), npad), 128, 0, ctx->stream>>>(summed(P, P->Sblk), summed(P, P->Scf), summed(P, P->Sff), summed(P, P->rhs), summed(P, P->dcf), P->nc, npad, 1.0 / radius,
                                                                                 opt->min_lm_diagonal, opt->max_lm_diagonal, P->A, st, P->solve_counter);
    SFM_LAUNCH_CHECK(ctx);
    const int ntasks = chol_stream_tasks(nbk);
    chol_stream_kernel<<<std::min(ntasks, P->chol_grid_stream), CS_THREADS, 0, ctx->stream>>>(P->A, npad, P->n, nbk, ntasks, P->dinv, P->fail + 1, P->chol_ready, P->chol_ll,
                                                                                          0u, P->Linv, nullptr, skip, P->solve_counter);
    SFM_LAUNCH_CHECK(ctx);
    if (P->backsolve_cluster) chol_backsolve_cluster_kernel<<<BS_CLUSTER, chol_backsolve_cluster_threads(P->n), chol_backsolve_cluster_smem(P->n), ctx->stream>>>(P->A, P->Linv, npad, P->n, P->y_cf, P->fail + 1, skip);
    else chol_backsolve_kernel<<<1, 640, chol_backsolve_smem(npad), ctx->stream>>>(P->A, P->Linv, npad, P->n, P->y_cf, skip);
    SFM_LAUNCH_CHECK(ctx);
    return SFMB200_OK;
}

// Host-side check of the flattened problem (CSR offsets monotone from 0 to nobs, cameras in range and strictly ascending
// inside a point = std::map order, reference :146).  It runs once per adjustBundle call over every observation, i.e. inside
// the end-to-end time of sfmb200_ba_solve (2 ms of a 17.7 ms cfg-3 solve when written as the obvious nested loop), so the
// common case is two flat, branch-free, vectorisable sweeps: range test over all cameras, and "descents" cam[o] <= cam[o-1]
// counted over all o against those that sit on a point boundary (where they are legal).  Only when a count is off does the
// slow loop run to name the offending element.
static int ba_validate_csr(int nc, int np, int nobs, const int32_t* obs_cam, const int32_t* pt_off, int* maxk_out, long long* pairs_out,
                           char* msg, size_t msg_len) {
    auto fail = [&](const char* fmt, int a, int b) { if (msg && msg_len) snprintf(msg, msg_len, fmt, a, b); return SFMB200_ERR_INVALID; };
    int maxk = 0; long long pairs = 0;
    if (maxk_out) *maxk_out = 0;
    if (pairs_out) *pairs_out = 0;
    if (np == 0) return nobs ? fail("observations without points (%d observations, %d points)", nobs, np) : SFMB200_OK;
    if (pt_off[0] != 0 || pt_off[np] != nobs) return fail("pt_off must start at 0 and end at nobs (%d .. %d)", pt_off[0], pt_off[np]);
    int neg = 0; long long boundary_descents = 0;
    for (int p = 0; p < np; ++p) {
        const int a = pt_off[p], b = pt_off[p + 1], k = b - a;
        neg |= k < 0;
        maxk = k > maxk ? k : maxk;
        pairs += (long long)k * (k - 1) / 2;
        // a descent across the boundary between the previous non-empty point and this one is legal
        if (k > 0 && a > 0 && a < nobs) boundary_descents += obs_cam[a] <= obs_cam[a - 1];
    }
    if (!neg) {
        unsigned out_of_range = nobs ? (unsigned)obs_cam[0] >= (unsigned)nc : 0u; long long descents = 0;
        for (int o = 1; o < nobs; ++o) { out_of_range |= (unsigned)obs_cam[o] >= (unsigned)nc; descents += obs_cam[o] <= obs_cam[o - 1]; }
        if (!out_of_range && descents == boundary_descents) {
            if (maxk_out) *maxk_out = maxk;
            if (pairs_out) *pairs_out = pairs;
            return SFMB200_OK;
        }
    }
    for (int p = 0; p < np; ++p) {              // something is wrong: find it
        if (pt_off[p + 1] < pt_off[p] || pt_off[p + 1] > nobs) return fail("pt_off not monotone within [0, nobs] at point %d (%d)", p, pt_off[p + 1]);
        for (int o = pt_off[p]; o < pt_off[p + 1]; ++o) {
            if (obs_cam[o] < 0 || obs_cam[o] >= nc) return fail("observation %d: camera %d out of range", o, obs_cam[o]);
            if (o > pt_off[p] && obs_cam[o] <= obs_cam[o - 1]) return fail("point %d: cameras must be strictly ascending (observation %d)", p, o);
        }
    }
    return fail("inconsistent observation lists (%d points, %d observations)", np, nobs);
}

extern "C" {

int sfmb200_ba_validate(int nc, int np, int nobs, const int32_t* obs_cam, const int32_t* pt_off, char* message, int message_len) {
    if (nc < 0 || np < 0 || nobs < 0 || (np && !pt_off) || (nobs && !obs_cam)) { if (message && message_len > 0) snprintf(message, message_len, "null buffer or negative size"); return SFMB200_ERR_INVALID; }
    int maxk = 0;
    int rc = ba_validate_csr(nc, np, nobs, obs_cam, pt_off, &maxk, nullptr, message, message_len > 0 ? (size_t)message_len : 0);
    if (rc == SFMB200_OK && maxk > 255) { if (message && message_len > 0) snprintf(message, message_len, "a point is observed by %d views; at most 255 supported", maxk); return SFMB200_ERR_UNSUPPORTED; }
    return rc;
}

void sfmb200_ba_default_options(sfmb200_ba_options* o) {
    if (!o) return;
    o->max_num_iterations = 500; o->max_solver_time_in_seconds = 10.0;
    o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
    o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32;
    o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32;
    o->jacobi_scaling = 1; o->max_num_consecutive_invalid_steps = 5; o->verbose = 0; o->profile = 0; o->l2_flush_mb = 0;
}

int sfmb200_ba_problem_create(sfmb200_ctx* ctx, int nc, int np, int nobs, const double* cams6, const double* pts3, double focal,
                              const float* obs_xy, const int32_t* obs_cam, const int32_t* pt_off, sfmb200_ba_problem** out) {
    if (!ctx || !out || nc < 0 || np < 0 || nobs < 0) return SFMB200_ERR_INVALID;
    *out = nullptr;
    if ((nc && !cams6) || (np && (!pts3 || !pt_off)) || (nobs && (!obs_xy || !obs_cam))) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "null buffer");
    // (the CSR is validated below, on the host, while the uploads are in flight)
    int maxk = 0; long long pair_entries = 0;

    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    sfmb200_ba_problem* P = new sfmb200_ba_problem();
    P->ctx = ctx; P->nc = nc; P->np = np; P->nobs = nobs;
    P->n = 6 * nc + 1; P->npad = ((P->n + 1) + NB - 1) / NB * NB;
    const size_t nblk = (size_t)nc * (nc + 1) / 2, n = P->n;
    P->red_n = 36 * nblk + 6 * (size_t)nc + 1 + 3 * n + 8;

    size_t bytes = 0;
    auto add = [&](size_t b) { bytes += Carver::pad(b) + 256; };
    add(8 * (size_t)nobs); add(4 * (size_t)nobs); add(4 * (size_t)(np + 1)); add(4 * (size_t)(nc + 1)); add(8 * (size_t)nobs); add(4 * (size_t)nobs);
    for (int i = 0; i < 3; ++i) { add(8 * n); add(24 * (size_t)np); }
    add(sizeof(CamDerived) * (size_t)nc); add(sizeof(CamDerived) * (size_t)nc);
    add(8 * n); add(24 * (size_t)np); add(8 * PTB * (size_t)np); add(8 * (P->red_n + 32));
    add(8 * (size_t)P->npad * P->npad); add(8 * n); add(8 * (size_t)P->npad); add(4 * (size_t)nobs); add(8 * (size_t)(nc + 1));
    add(4 * (size_t)(P->npad / NB) * (P->npad / NB)); add(8 * (size_t)P->npad * NB); add(chol_ll_bytes(P->npad / NB)); add(sizeof(LMState));
    add(4 * (size_t)nobs); add((size_t)nobs); add(8 * 4 * (size_t)ctx->sm_count * 32); add(16 * (size_t)(nc + 1)); add(64);   // cm_obs, cm_np, part4, fpart, counters
    if (!ctx->ba_ws.in_use) {           // borrow the cached workspace (grown below when too small)
        P->mem = ctx->ba_ws.mem; P->gmem = ctx->ba_ws.gmem; P->xbuf = ctx->ba_ws.xbuf; P->hpin = ctx->ba_ws.hpin;
        ctx->ba_ws.mem = DevBuf(); ctx->ba_ws.gmem = DevBuf(); ctx->ba_ws.xbuf = DevBuf(); ctx->ba_ws.hpin = PinBuf();
        ctx->ba_ws.in_use = true; P->borrowed = true;
    }
    cudaError_t e = P->mem.reserve(bytes);
    if (e != cudaSuccess) { ba_release_buffers(P); delete P; return sfmb200_fail(ctx, SFMB200_ERR_NOMEM, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); }
    Carver cv(P->mem.p);
    P->obs_xy = cv.take<float2>(nobs); P->obs_cam = cv.take<int32_t>(nobs); P->pt_off = cv.take<int32_t>(np + 1); P->cm_off = cv.take<int32_t>(nc + 1);
    P->cm_xy = cv.take<float2>(nobs); P->cm_pt = cv.take<int32_t>(nobs);
    P->cf[0] = cv.take<double>(n); P->pts[0] = cv.take<double>(3 * (size_t)np); P->cf[1] = cv.take<double>(n); P->pts[1] = cv.take<double>(3 * (size_t)np);
    P->cf0 = cv.take<double>(n); P->pts0 = cv.take<double>(3 * (size_t)np);
    P->camd[0] = cv.take<CamDerived>(nc); P->camd[1] = cv.take<CamDerived>(nc);
    P->scale_cf = cv.take<double>(n); P->scale_pt = cv.take<double>(3 * (size_t)np); P->ptblk = cv.take<double>(PTB * (size_t)np);
    // exchange memory: [red (red_n) | locals 8 | gmax 1 | pad 1 | fail 1 | pad 1 | post 8 | pad 4][flags 2*MAX_PEERS u64]
    P->xmem_doubles = P->red_n + 24 + 2 * MAX_PEERS;
    {
        cudaError_t ex = P->xbuf.reserve(8 * P->xmem_doubles + 256);
        if (ex != cudaSuccess) { ba_release_buffers(P); delete P; return sfmb200_fail(ctx, SFMB200_ERR_NOMEM, "cudaMalloc(exchange): %s", cudaGetErrorString(ex)); }
        P->xmem = P->xbuf.p;
        cudaMemsetAsync(P->xmem, 0, 8 * P->xmem_doubles + 256, ctx->stream);
    }
    P->red = (double*)P->xmem;
    P->xtmp = cv.take<double>(P->red_n + 32);
    P->Sblk = P->red; P->Scf = P->Sblk + 36 * nblk; P->Sff = P->Scf + 6 * (size_t)nc; P->rhs = P->Sff + 1; P->gcf = P->rhs + n; P->dcf = P->gcf + n; P->sums = P->dcf + n;
    // after red: locals 8 | gmax 1 | pad 1 | fail 1 | pad 1 | post 8 | pad 4 | flags
    P->locals = P->red + P->red_n; P->gmax_pt_bits = (unsigned long long*)(P->locals + 8); P->fail = (int*)(P->locals + 10); P->post = P->locals + 12;
    P->xflags = (unsigned long long*)(P->red + P->red_n + 24);
    P->A = cv.take<double>((size_t)P->npad * P->npad); P->y_cf = cv.take<double>(n); P->dinv = cv.take<double>(P->npad);
    int32_t* obs_pt = cv.take<int32_t>(nobs); int* cnt = cv.take<int>(2 * (size_t)(nc + 1)); int* cursor = cnt + nc + 1;
    P->obs_pt = obs_pt; P->cm_obs = cv.take<int32_t>(nobs); P->cm_np = cv.take<uint8_t>(nobs);
    P->part4 = cv.take<double>(4 * (size_t)ctx->sm_count * 32); P->fpart = cv.take<double>(2 * (size_t)(nc + 1)); P->counters = cv.take<unsigned>(16);
    P->solve_counter = P->counters + 8;
    P->chol_ready = cv.take<unsigned>((size_t)(P->npad / NB) * (P->npad / NB));
    P->Linv = cv.take<double>((size_t)P->npad * NB);
    P->chol_ll = cv.take<uint4>(chol_ll_bytes(P->npad / NB) / sizeof(uint4));
    P->d_state = cv.take<LMState>(1);

    cudaStream_t st = ctx->stream;
#define CRT(call) do { cudaError_t e2 = (call); if (e2 != cudaSuccess) { ba_release_buffers(P); delete P; return sfmb200_fail(ctx, SFMB200_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e2)); } } while (0)
    if (nobs) { CRT(cudaMemcpyAsync(P->obs_xy, obs_xy, 8 * (size_t)nobs, cudaMemcpyHostToDevice, st)); CRT(cudaMemcpyAsync(P->obs_cam, obs_cam, 4 * (size_t)nobs, cudaMemcpyHostToDevice, st)); }
    if (np) { CRT(cudaMemcpyAsync(P->pt_off, pt_off, 4 * (size_t)(np + 1), cudaMemcpyHostToDevice, st)); CRT(cudaMemcpyAsync(P->pts0, pts3, 24 * (size_t)np, cudaMemcpyHostToDevice, st)); }
    if (nc) CRT(cudaMemcpyAsync(P->cf0, cams6, 48 * (size_t)nc, cudaMemcpyHostToDevice, st));
    P->focal0 = focal;                  // the copy source must outlive this stack frame's uses: a member
    CRT(cudaMemcpyAsync(P->cf0 + 6 * nc, &P->focal0, 8, cudaMemcpyHostToDevice, st));
    {   // validate the CSR while the uploads run: offsets monotone, cameras in range and strictly ascending within a point
        // (std::map order, :146).  Nothing that indexes by camera or offset is launched before this passes.
        char msg[160]; msg[0] = 0;
        int vrc = ba_validate_csr(nc, np, nobs, obs_cam, pt_off, &maxk, &pair_entries, msg, sizeof msg);
        if (vrc == SFMB200_OK && maxk > 255) { snprintf(msg, sizeof msg, "a point is observed by %d views; at most 255 supported", maxk); vrc = SFMB200_ERR_UNSUPPORTED; }
        if (vrc == SFMB200_OK) {
            P->maxk = std::max(maxk, 1);
            P->G = maxk <= 4 ? 4 : maxk <= 8 ? 8 : maxk <= 16 ? 16 : 32;
            if (point_smem_bytes(P->G, P->maxk) > 200 * 1024) { snprintf(msg, sizeof msg, "observations per point (%d) exceed the shared-memory budget", maxk); vrc = SFMB200_ERR_UNSUPPORTED; }
        }
        if (vrc != SFMB200_OK) { cudaStreamSynchronize(st); ba_release_buffers(P); delete P; return sfmb200_fail(ctx, vrc, "%s", msg); }
    }
    // camera-major copy (device counting sort)
    CRT(cudaMemsetAsync(cnt, 0, sizeof(int) * 2 * (nc + 1), st));
    {   // dataflow Cholesky: ready flags start at epoch 0; the grid must stay within the co-resident CTA count
        const int nbk = P->npad / NB;
        CRT(cudaMemsetAsync(P->chol_ready, 0, 4 * (size_t)nbk * nbk, st));
        CRT(cudaMemsetAsync(P->chol_ll, 0, chol_ll_bytes(nbk), st));
        int per_sm = 0;
        CRT(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chol_stream_kernel, CS_THREADS, 0));
        if (per_sm < 1) {
            cudaStreamSynchronize(st); ba_release_buffers(P); delete P;
            return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "the dense Cholesky kernel cannot be resident on this device");
        }
        P->chol_grid_stream = per_sm * ctx->sm_count;
        // back substitution on a cluster of BS_CLUSTER SMs while its per-CTA slices fit (n <= 2816, 469 cameras), on one CTA above
        const size_t cs = chol_backsolve_cluster_smem(P->n);
        P->backsolve_cluster = cs <= 200 * 1024 && chol_backsolve_cluster_threads(P->n) <= 512;
        if (P->backsolve_cluster) CRT(cudaFuncSetAttribute(chol_backsolve_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs));
    }
    CRT(cudaMemsetAsync(P->counters, 0, 64, st));
    {   // mode: gather (default: ba_pair_kernel + ba_combine_kernel, deterministic) needs the pair-list fill's per-warp camera counters in shared
        // memory and the stable sort's per-warp counters; "red" (SFMB200_BA_SCHUR=red, or too many cameras) uses atomics
        const char* mode = getenv("SFMB200_BA_SCHUR");
        // partial blocks of the pair kernel: one 288-byte block per (camera pair, point segment[, split]); with thousands of cameras
        // that buffer (and the per-key offset tables) outgrow their use -- such problems take the atomics path
        const size_t nseg_est = (size_t)pair_segments(ctx, nobs);
        const bool partials_fit = nblk * nseg_est * 288 <= ((size_t)256 << 20);
        P->gather = !(mode && strcmp(mode, "red") == 0) && (size_t)(2 * PFILL_WARPS + 1) * nc * 4 <= 160 * 1024 && pair_entries < (1LL << 31) - 1024 && partials_fit;
    }
    if (nobs) {
        expand_obs_pt_kernel<<<ceil_div(np, 256), 256, 0, st>>>(P->pt_off, np, obs_pt);
        ctx->launches += 1;
    }
    if (nobs && P->gather) {
        // stable counting sort by camera (no arrival-order atomics): per-CTA histograms, per-camera scan over the CTAs, scatter
        const int ncta = ceil_div(nobs, CMS_THREADS);
        const size_t hist_bytes = Carver::pad(4 * (size_t)ncta * nc);
        const size_t smem = sizeof(int) * (size_t)CMS_WARPS * nc;
        // geometry of the camera-major kernel: one balanced wave of slices; partial records (slices + cameras)
        const size_t fill_smem = sizeof(int) * (size_t)(2 * PFILL_WARPS + 1) * nc;
        if (smem > 48 * 1024) {
            CRT(cudaFuncSetAttribute(cm_sort_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            CRT(cudaFuncSetAttribute(cm_sort_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        }
        if (fill_smem > 48 * 1024) CRT(cudaFuncSetAttribute(pair_fill_sorted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fill_smem));
        {
            int per_sm = 0;
            CRT(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ba_camera_kernel<true, false>, CAM_THREADS, 0));
            P->diag_grid = std::max(1, std::min(ceil_div(nobs, CAM_THREADS), std::max(1, per_sm) * ctx->sm_count));
            P->diag_per_cta = ceil_div(nobs, P->diag_grid);
            P->diag_grid = ceil_div(nobs, P->diag_per_cta);
        }
        // off-diagonal blocks: per-(camera pair, point segment) entry lists, one segment of Zbuf small enough to stay L2-resident
        // while it is read ~7 times (pair_segments); one partial block per (pair, segment, split) warp
        const long long E = pair_entries;           // observation pairs of a point, counted by the validation sweep
        const int nseg = pair_segments(ctx, nobs);
        const size_t nkeys = nblk * (size_t)nseg;
        // splits are fixed before the lists exist (they size the partial buffer): assume every pair is non-empty
        P->pair_nseg = nseg;
        P->pair_splits = std::max(1, std::min(64, ceil_div(16 * ctx->sm_count, (int)std::max<size_t>(1, nblk - nc))));
        // ...but a list is not worth splitting below ~64 entries per warp (tiny problems: 64 splits of a 100-entry list made the
        // combine kernel the longest of the iteration)
        P->pair_splits = (int)std::max<long long>(1, std::min<long long>(P->pair_splits, E / (64 * (long long)std::max<size_t>(1, (nblk - nc) * (size_t)nseg))));
        const size_t part_bytes = Carver::pad(8 * (size_t)(P->diag_grid + nc) * ROW_HDR) + Carver::pad(8 * 36 * nkeys * P->pair_splits);
        const size_t gb = Carver::pad(8 * 18 * (size_t)nobs) + part_bytes + hist_bytes + Carver::pad(4 * (nkeys + 1)) + Carver::pad(4 * (nblk + 1)) +
                          Carver::pad(8 * (size_t)std::max<long long>(E, 1)) + Carver::pad(4 * nkeys) * 2 + 8192;
        CRT(P->gmem.reserve(gb));
        Carver gc(P->gmem.p);
        P->Zbuf = gc.take<double>(18 * (size_t)nobs);
        P->diag_part = gc.take<double>((size_t)(P->diag_grid + nc) * ROW_HDR);
        P->pair_part = gc.take<double>(36 * nkeys * P->pair_splits);
        P->pair_off = gc.take<int32_t>(nkeys + 1); P->pair_blk = gc.take<int32_t>(nblk + 1);
        P->pair_ent = gc.take<uint2>((size_t)std::max<long long>(E, 1));
        int* pcnt = gc.take<int>(nkeys); int* pcur = gc.take<int>(nkeys); int* d_nne = gc.take<int>(4);
        int* hist = gc.take<int>((size_t)ncta * nc);
        cm_sort_kernel<false><<<ncta, CMS_THREADS, smem, st>>>(P->obs_cam, P->obs_xy, obs_pt, P->pt_off, nobs, nc, hist, nullptr, nullptr, nullptr, nullptr, nullptr);
        cm_scan_ctas_kernel<<<nc, 1024, 0, st>>>(hist, ncta, nc, cnt);
        scan_small_kernel<<<1, 32, 0, st>>>(cnt, nc, P->cm_off, cursor);
        cm_sort_kernel<true><<<ncta, CMS_THREADS, smem, st>>>(P->obs_cam, P->obs_xy, obs_pt, P->pt_off, nobs, nc, hist, P->cm_off, P->cm_xy, P->cm_pt, P->cm_obs, P->cm_np);
        ctx->launches += 4;
        if (E > 0) {
            CRT(cudaMemsetAsync(pcnt, 0, 4 * nkeys, st));
            pair_count_kernel<<<ceil_div(np, 256), 256, 0, st>>>(P->pt_off, P->obs_cam, np, nc, nseg, pcnt);
            pair_scan_kernel<<<1, 1024, 0, st>>>(pcnt, (int)nkeys, P->pair_off, pcur);
            pair_compact_kernel<<<1, 1024, 0, st>>>(P->pair_off, (int)nblk, nseg, P->pair_blk, d_nne);
            pair_fill_sorted_kernel<<<nc, PFILL_THREADS, fill_smem, st>>>(P->cm_off, P->cm_obs, P->cm_np, P->obs_cam, nc, nseg, P->pair_off, P->pair_ent);
            ctx->launches += 4;
            CRT(cudaGetLastError());
            int nne = 0;
            CRT(cudaMemcpyAsync(&nne, d_nne, 4, cudaMemcpyDeviceToHost, st));
            CRT(cudaStreamSynchronize(st));
            P->n_pairs_nonempty = nne;
        } else {
            CRT(cudaMemsetAsync(P->pair_off, 0, 4 * (nkeys + 1), st));
        }
    } else if (nobs) {
        const int use_smem = (size_t)nc * 8 <= 40 * 1024;
        count_cams_kernel<<<ceil_div(nobs, SORT_THREADS), SORT_THREADS, use_smem ? nc * 4 : 0, st>>>(P->obs_cam, nobs, nc, use_smem, cnt);
        scan_small_kernel<<<1, 32, 0, st>>>(cnt, nc, P->cm_off, cursor);
        scatter_cm_kernel<<<ceil_div(nobs, SORT_THREADS), SORT_THREADS, use_smem ? nc * 8 : 0, st>>>(P->obs_cam, P->obs_xy, obs_pt, nobs, nc, use_smem, cursor, P->cm_xy, P->cm_pt);
        ctx->launches += 3;
    } else {
        scan_small_kernel<<<1, 32, 0, st>>>(cnt, nc, P->cm_off, cursor); ctx->launches += 1;
    }
    CRT(cudaGetLastError());
    CRT(P->hpin.reserve(sizeof(double) * 32 + sizeof(LMState))); P->h_scal = (double*)P->hpin.p; P->h_state = (LMState*)(P->h_scal + 32);
    {
        if (P->gather && !P->Zbuf) {     // no observations: a dummy Z buffer keeps the kernels' pointers valid
            CRT(P->gmem.reserve(Carver::pad(8 * 18) + 256));
            P->Zbuf = (double*)P->gmem.p;
        }
        const char* bm = getenv("SFMB200_BA_BACKSUB");
        // Z blocks when all of Zbuf is one L2-sized pair segment (still L2-resident from the point pass, and the 64-register
        // kernel fits a small problem in one wave); otherwise re-evaluated Jacobians save the 144-byte record per observation
        // that would come from HBM.  SFMB200_BA_BACKSUB=stored / jacobian forces either.
        const bool z_in_l2 = P->pair_nseg == 1;
        P->backsub_from_z = P->gather && P->Zbuf && (bm ? strcmp(bm, "stored") == 0 : z_in_l2);
    }
#undef CRT
    *out = P;
    SFM_CUDA(ctx, cudaMemcpyAsync(P->cf[0], P->cf0, 8 * n, cudaMemcpyDeviceToDevice, st));
    if (np) SFM_CUDA(ctx, cudaMemcpyAsync(P->pts[0], P->pts0, 24 * (size_t)np, cudaMemcpyDeviceToDevice, st));
    P->cur = 0; P->have_scale = false; P->camd_valid[0] = P->camd_valid[1] = false;
    SFM_CUDA(ctx, cudaStreamSynchronize(st));
    return SFMB200_OK;
}

void sfmb200_ba_problem_destroy(sfmb200_ba_problem* P) {
    if (!P) return;
    std::lock_guard<std::mutex> lk(P->ctx->mu);
    cudaSetDevice(P->ctx->device);
    cudaStreamSynchronize(P->ctx->stream);
    for (int k = 0; k < LM_CHUNK_MAX; ++k) for (int e = 0; e < 8; ++e) if (P->evs[k].ev[e]) cudaEventDestroy(P->evs[k].ev[e]);
    // peer mappings stay open in the context's cache (ctx->ipc_cache) for the next problem; closed with the context
    ba_release_buffers(P);
    delete P;
}

int sfmb200_ba_problem_reset(sfmb200_ba_problem* P) {
    if (!P) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = P->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    SFM_CUDA(ctx, cudaMemcpyAsync(P->cf[0], P->cf0, 8 * (size_t)P->n, cudaMemcpyDeviceToDevice, ctx->stream));
    if (P->np) SFM_CUDA(ctx, cudaMemcpyAsync(P->pts[0], P->pts0, 24 * (size_t)P->np, cudaMemcpyDeviceToDevice, ctx->stream));
    P->cur = 0; P->have_scale = false; P->camd_valid[0] = P->camd_valid[1] = false;
    return SFMB200_OK;
}

int sfmb200_ba_problem_download(sfmb200_ba_problem* P, double* cams6, double* pts3, double* focal) {
    if (!P) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = P->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    if (cams6 && P->nc) SFM_CUDA(ctx, cudaMemcpyAsync(cams6, P->cf[P->cur], 48 * (size_t)P->nc, cudaMemcpyDeviceToHost, ctx->stream));
    if (focal) SFM_CUDA(ctx, cudaMemcpyAsync(focal, P->cf[P->cur] + 6 * P->nc, 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (pts3 && P->np) SFM_CUDA(ctx, cudaMemcpyAsync(pts3, P->pts[P->cur], 24 * (size_t)P->np, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SFMB200_OK;
}

int sfmb200_ba_problem_ipc_handle(sfmb200_ba_problem* P, uint8_t* out) {
    if (!P || !out) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = P->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    static_assert(sizeof(h) == SFMB200_IPC_HANDLE_BYTES, "IPC handle size");
    SFM_CUDA(ctx, cudaIpcGetMemHandle(&h, P->xmem));
    memcpy(out, &h, sizeof h);
    return SFMB200_OK;
}

static int ba_attach_handles(sfmb200_ba_problem* P, const uint8_t* handles);

int sfmb200_ba_problem_ipc_attach(sfmb200_ba_problem* P, const uint8_t* handles) {
    if (!P) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = P->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    return ba_attach_handles(P, handles);
}

}  // extern "C"

static int ba_attach_handles(sfmb200_ba_problem* P, const uint8_t* handles) {
    sfmb200_ctx* ctx = P->ctx;
    if (ctx->nranks <= 1) return SFMB200_OK;
    if (!handles) return sfmb200_fail(ctx, SFMB200_ERR_INVALID, "handles required");
    if (ctx->nranks > MAX_PEERS) return sfmb200_fail(ctx, SFMB200_ERR_UNSUPPORTED, "at most %d ranks", MAX_PEERS);
    for (int r = 0; r < ctx->nranks; ++r) {
        void* base = P->xmem;
        if (r != ctx->rank) {
            std::array<uint8_t, 64> key; memcpy(key.data(), handles + (size_t)r * SFMB200_IPC_HANDLE_BYTES, 64);
            base = nullptr;
            for (auto& e : ctx->ipc_cache) if (e.first == key) { base = e.second; break; }
            if (!base) {
                cudaIpcMemHandle_t h; memcpy(&h, key.data(), sizeof h);
                cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
                if (e != cudaSuccess) return sfmb200_fail(ctx, SFMB200_ERR_COMM, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
                ctx->ipc_cache.push_back({key, base});
            }
            P->peer_base[r] = base;
        }
        P->ptab.buf[r] = (double*)base;
        P->ptab.flags[r] = (unsigned long long*)((double*)base + P->red_n + 24);
    }
    P->peers = true;
    return SFMB200_OK;
}

// The one-shot solve attaches its peers itself: export this problem's exchange buffer, all-gather the 64-byte CUDA-IPC handles
// over the library's NCCL communicator (the only NCCL call of the solve), map the peers (mappings are cached in the context).
// SFMB200_EXCHANGE=nccl keeps the NCCL all-reduce data path.  ctx->mu is held.
static int ba_auto_attach(sfmb200_ba_problem* P) {
    sfmb200_ctx* ctx = P->ctx;
    if (ctx->nranks <= 1 || P->peers) return SFMB200_OK;
    const char* ex = getenv("SFMB200_EXCHANGE");
    if (ex && strcmp(ex, "nccl") == 0) return SFMB200_OK;
    if (ctx->nranks > MAX_PEERS) return SFMB200_OK;
    cudaIpcMemHandle_t h;
    SFM_CUDA(ctx, cudaIpcGetMemHandle(&h, P->xmem));
    const size_t nb = SFMB200_IPC_HANDLE_BYTES;
    SFM_CUDA(ctx, ctx->scratch.reserve(nb * (ctx->nranks + 1) + 256));
    uint8_t* d_send = (uint8_t*)ctx->scratch.p; uint8_t* d_recv = d_send + 256;
    SFM_CUDA(ctx, cudaMemcpyAsync(d_send, &h, nb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = sfmb200_allgather_bytes(ctx, d_send, d_recv, nb); if (rc) return rc;
    std::vector<uint8_t> all(nb * ctx->nranks);
    SFM_CUDA(ctx, cudaMemcpyAsync(all.data(), d_recv, all.size(), cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return ba_attach_handles(P, all.data());
}

extern "C" {

int sfmb200_ba_problem_reduced_system(sfmb200_ba_problem* P, const sfmb200_ba_options* opt_in, double radius,
                                      double* S, double* rhs, double* grad_cf, double* cost) {
    if (!P || !(radius > 0)) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = P->ctx;
    sfmb200_ba_options opt; if (opt_in) opt = *opt_in; else sfmb200_ba_default_options(&opt);
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if (!P->have_scale) { rc = compute_scaling(P, &opt); if (rc) return rc; }
    rc = schur_pass(P, &opt, radius, nullptr, false); if (rc) return rc;
    const int n = P->n, npad = P->npad;
    ba_assemble_kernel<<<dim3(ceil_div(npad, 128), npad), 128, 0, ctx->stream>>>(summed(P, P->Sblk), summed(P, P->Scf), summed(P, P->Sff), summed(P, P->rhs), summed(P, P->dcf), P->nc, npad, 1.0 / radius,
                                                                                 opt.min_lm_diagonal, opt.max_lm_diagonal, P->A, nullptr, nullptr);
    SFM_LAUNCH_CHECK(ctx);
    std::vector<double> hA((size_t)npad * npad), hg(n), hs(n), hsum(8);
    SFM_CUDA(ctx, cudaMemcpyAsync(hA.data(), P->A, 8 * hA.size(), cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(hg.data(), summed(P, P->gcf), 8 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(hs.data(), P->scale_cf, 8 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    SFM_CUDA(ctx, cudaMemcpyAsync(hsum.data(), summed(P, P->sums), 64, cudaMemcpyDeviceToHost, ctx->stream));
    rc = ba_peer_barrier(P); if (rc) return rc;
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (S) for (int r = 0; r < n; ++r) for (int c = 0; c <= r; ++c) { const double v = hA[(size_t)r * npad + c]; S[(size_t)r * n + c] = v; S[(size_t)c * n + r] = v; }
    if (rhs) for (int c = 0; c < n; ++c) rhs[c] = hA[(size_t)n * npad + c];
    if (grad_cf) for (int c = 0; c < n; ++c) grad_cf[c] = hg[c] / hs[c];
    if (cost) *cost = 0.5 * hsum[0];
    return SFMB200_OK;
}

// The LM loop.  Control state lives on the device (LMState, ba_lm_control_kernel); the host enqueues LM_CHUNK complete
// iterations at a time -- pass, rank sum, dense solve, candidate, evaluation, rank sum, control -- and reads the state back
// once per chunk: no stream synchronisation, read-back or host decision inside a chunk, and the next chunk's launches are
// issued while the GPU is still working when the solve continues.  An iteration enqueued after the solve has terminated is a
// no-op (every kernel checks LMState::status first).  Only the wall-clock limit is tested on the host, between chunks.
int sfmb200_ba_problem_run(sfmb200_ba_problem* P, const sfmb200_ba_options* opt_in, sfmb200_ba_summary* sum) {
    if (!P || !sum) return SFMB200_ERR_INVALID;
    sfmb200_ctx* ctx = P->ctx;
    sfmb200_ba_options opt; if (opt_in) opt = *opt_in; else sfmb200_ba_default_options(&opt);
    std::lock_guard<std::mutex> lk(ctx->mu);
    SFM_CUDA(ctx, cudaSetDevice(ctx->device));
    memset(sum, 0, sizeof *sum);
    const auto t_start = std::chrono::steady_clock::now();
    auto elapsed = [&]() { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count(); };
    const int64_t launches0 = ctx->launches;
    int rc = compute_scaling(P, &opt); if (rc) return rc;
    if (opt.profile && !P->have_events) {
        for (int k = 0; k < LM_CHUNK_MAX; ++k) for (int e = 0; e < 8; ++e) SFM_CUDA(ctx, cudaEventCreate(&P->evs[k].ev[e]));
        P->have_events = true;
    }
    if (!P->camd_valid[P->cur]) {       // inside the loop the table of an accepted candidate comes from ba_cam_update_kernel
        cam_derive_kernel<<<ceil_div(std::max(1, P->nc), 128), 128, 0, ctx->stream>>>(P->cf[P->cur], P->nc, P->camd[P->cur]); SFM_LAUNCH_CHECK(ctx);
        P->camd_valid[P->cur] = true;
    }
    LMState* hs = P->h_state;
    memset(hs, 0, sizeof *hs);
    hs->radius = opt.initial_trust_region_radius; hs->decrease_factor = 2.0; hs->cur = P->cur; hs->new_point = 1;
    hs->status = LM_RUNNING; hs->termination_type = SFMB200_BA_NO_CONVERGENCE;
    SFM_CUDA(ctx, cudaMemcpyAsync(P->d_state, hs, sizeof *hs, cudaMemcpyHostToDevice, ctx->stream));
    SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                 // hs is reused for the read-back
    const int chunk_default = P->nobs < 100000 ? LM_CHUNK_MAX : LM_CHUNK;
    int chunk = opt.verbose ? 1 : chunk_default;
    if (const char* ce = getenv("SFMB200_BA_CHUNK")) chunk = std::max(1, std::min(LM_CHUNK_MAX, atoi(ce)));
    bool timed_out = false;
    int executed = 0;
    // Multi-GPU: every rank must enqueue the SAME sequence of exchanges, so nothing rank-local may decide when the loop stops.
    // The LM decisions are identical by construction (rank-summed inputs); the wall-clock limit is not -- each rank's flag
    // "my clock says stop" is max-reduced over the ranks at the end of every chunk and all ranks act on the result.  The chunk
    // size must be the same everywhere too: options (verbose) must match across ranks, the environment override is ignored.
    const bool collective_clock = ctx->nranks > 1 && opt.max_solver_time_in_seconds > 0;
    if (ctx->nranks > 1) chunk = opt.verbose ? 1 : LM_CHUNK;       // (per-rank shard sizes differ: no size-dependent choice here)
    double* tflag = P->post + 8;      // one of the pad doubles behind post[8] in the exchange buffer

    // one LM iteration on the device: pass at x, dense solve, candidate, evaluation, decision
    auto enqueue_iteration = [&](const EvSet* es) -> int {
        if (opt.l2_flush_mb > 0) {      // benchmark hygiene: evict the working set from L2 between iterations
            SFM_CUDA(ctx, ctx->scratch2.reserve((size_t)opt.l2_flush_mb << 20));
            if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[6], ctx->stream));
            SFM_CUDA(ctx, cudaMemsetAsync(ctx->scratch2.p, 0, (size_t)opt.l2_flush_mb << 20, ctx->stream));
            if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[7], ctx->stream));
        }
        int r = schur_pass(P, &opt, 0.0, es, true); if (r) return r;
        if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[4], ctx->stream));
        r = dense_solve(P, &opt, 0.0, true); if (r) return r;
        if (es) SFM_CUDA(ctx, cudaEventRecord(es->ev[5], ctx->stream));
        BAView v = make_view(P, &opt, true);
        {
            BAView vc = v; vc.dcf = summed(P, P->dcf);              // the rank-summed J^T J diagonal and gradient
            ba_cam_update_kernel<<<1, 256, 0, ctx->stream>>>(vc, 0.0, nullptr, P->y_cf, P->scale_cf, summed(P, P->gcf), P->nc, nullptr, nullptr, P->locals,
                                                             P->post, P->gmax_pt_bits, P->fail);
        }
        SFM_LAUNCH_CHECK(ctx);
        if (P->np > 0 && P->nobs > 0) { r = DISPATCH_G(P, launch_backsub)(P, v); if (r) return r; }
        r = ba_allreduce(P, P->post, 7, 1); if (r) return r;   // sums: candidate cost, model, norms, failure counts; max: |g| of the points
        ba_lm_control_kernel<<<1, 32, 0, ctx->stream>>>(P->d_state, summed(P, P->sums), summed(P, P->post), P->locals, opt); SFM_LAUNCH_CHECK(ctx);
        return SFMB200_OK;
    };
    // Small problems (adjustBundle inside runSfM: hundreds to a few thousand observations, up to ~100 iterations) are bound by the
    // host's launch rate -- ~14 launches of microsecond kernels per iteration.  After a first ordinary chunk the remaining
    // iterations are replayed from a CUDA graph of GRAPH_ITERS iterations (one launch per replay; every kernel takes x, the
    // radius, the early-out and the dense-solve number from device memory, so frozen arguments are fine).  Single GPU, no
    // profiling / flushing / verbose output; SFMB200_BA_GRAPH=0 disables it.
    constexpr int GRAPH_ITERS = 8, GRAPH_AFTER = 4;      // the first ordinary chunk also warms every code path; solves that end inside it never build a graph
    const char* genv = getenv("SFMB200_BA_GRAPH");
    const bool graph_ok = ctx->nranks == 1 && !opt.profile && opt.l2_flush_mb <= 0 && !opt.verbose && P->gather && P->nobs < 100000 &&
                          !(genv && genv[0] == '0');
    if (graph_ok) chunk = std::min(chunk, LM_CHUNK);
    cudaGraphExec_t gexec = nullptr;
    int64_t graph_launches = 0;
    struct GraphGuard { cudaGraphExec_t* g; ~GraphGuard() { if (*g) cudaGraphExecDestroy(*g); } } graph_guard{&gexec};

    for (;;) {
        if (!collective_clock && executed > 0 && opt.max_solver_time_in_seconds > 0 && elapsed() >= opt.max_solver_time_in_seconds) { timed_out = true; break; }
        int n_it = std::max(1, std::min(chunk, opt.max_num_iterations - hs->iter));
        if (graph_ok && executed >= GRAPH_AFTER) {
            if (!gexec) {
                const int64_t l0 = ctx->launches;
                cudaGraph_t graph = nullptr;
                SFM_CUDA(ctx, cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
                int crc = SFMB200_OK;
                for (int k = 0; k < GRAPH_ITERS && crc == SFMB200_OK; ++k) crc = enqueue_iteration(nullptr);
                if (crc == SFMB200_OK && cudaMemcpyAsync(hs, P->d_state, sizeof *hs, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) crc = SFMB200_ERR_CUDA;
                const cudaError_t ce = cudaStreamEndCapture(ctx->stream, &graph);
                if (crc != SFMB200_OK || ce != cudaSuccess) { if (graph) cudaGraphDestroy(graph); return crc ? crc : sfmb200_fail(ctx, SFMB200_ERR_CUDA, "graph capture: %s", cudaGetErrorString(ce)); }
                const cudaError_t ie = cudaGraphInstantiate(&gexec, graph, 0);
                cudaGraphDestroy(graph);
                if (ie != cudaSuccess) return sfmb200_fail(ctx, SFMB200_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ie));
                graph_launches = ctx->launches - l0;                      // counted while capturing: subtract, add per replay
                ctx->launches = l0;
            }
            n_it = GRAPH_ITERS;
            SFM_CUDA(ctx, cudaGraphLaunch(gexec, ctx->stream));
            ctx->launches += graph_launches;
        } else {
            for (int k = 0; k < n_it; ++k) { rc = enqueue_iteration(opt.profile ? &P->evs[k] : nullptr); if (rc) return rc; }
        }
        if (collective_clock) {
            P->h_scal[30] = elapsed() >= opt.max_solver_time_in_seconds ? 1.0 : 0.0;
            SFM_CUDA(ctx, cudaMemcpyAsync(tflag, P->h_scal + 30, 8, cudaMemcpyHostToDevice, ctx->stream));
            rc = ba_allreduce(P, tflag, 0, 1); if (rc) return rc;
            SFM_CUDA(ctx, cudaMemcpyAsync(P->h_scal + 31, summed(P, tflag), 8, cudaMemcpyDeviceToHost, ctx->stream));
        }
        if (!gexec) SFM_CUDA(ctx, cudaMemcpyAsync(hs, P->d_state, sizeof *hs, cudaMemcpyDeviceToHost, ctx->stream));   // (part of the graph otherwise)
        SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        // iterations of this chunk that actually ran: all of them unless the solve terminated inside the chunk
        const int ran = hs->status == LM_RUNNING ? n_it : std::max(1, std::min(n_it, hs->passes - executed));
        executed += ran;
        if (opt.profile) {
            for (int k = 0; k < ran; ++k) {
                const EvSet& es = P->evs[k];
                float ms = 0;
                if (opt.l2_flush_mb > 0 && cudaEventElapsedTime(&ms, es.ev[6], es.ev[7]) == cudaSuccess) sum->flush_ms_total += ms;
                if (cudaEventElapsedTime(&ms, es.ev[4], es.ev[5]) == cudaSuccess) sum->solve_ms_total += ms;
                if (P->np > 0 && P->nobs > 0) {
                    if (cudaEventElapsedTime(&ms, es.ev[0], es.ev[1]) == cudaSuccess) { sum->schur_ms_total += ms; sum->schur_launches++; }
                    if (P->gather && cudaEventElapsedTime(&ms, es.ev[1], es.ev[2]) == cudaSuccess) { sum->pair_ms_total += ms; sum->pair_launches++; }
                    if (cudaEventElapsedTime(&ms, es.ev[2], es.ev[3]) == cudaSuccess) sum->camera_ms_total += ms;
                }
            }
        }
        if (opt.verbose) printf("iter %3d cost %.9e |g|max %.3e radius %.3e rho %.3e %s\n", hs->iter, hs->x_cost, hs->gmax, hs->radius, hs->last_rho,
                                hs->status != LM_RUNNING ? "stop" : (hs->new_point ? "ok" : "rejected"));
        if (hs->status != LM_RUNNING) break;
        if (collective_clock && P->h_scal[31] != 0.0) { timed_out = true; break; }
    }
    // final hand-shake of the peer exchange: after it no rank reads this rank's exchange buffer any more, so the caller may
    // destroy the problem (the buffer goes back to the workspace cache, is cleared by the next create, or is freed)
    rc = ba_peer_barrier(P); if (rc) return rc;
    if (P->peers) SFM_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    P->cur = hs->cur;
    P->camd_valid[P->cur] = true; P->camd_valid[P->cur ^ 1] = false;
    sum->termination_type = hs->termination_type;
    sum->num_iterations = hs->iter; sum->num_successful_steps = hs->num_successful; sum->num_unsuccessful_steps = hs->num_unsuccessful;
    sum->num_jacobian_passes = executed; sum->num_linear_solves = executed;
    sum->initial_cost = hs->initial_cost; sum->final_cost = hs->x_cost;
    const int why = timed_out ? LM_MAX_TIME : hs->status;
    switch (why) {
        case LM_EVAL_FAILED: snprintf(sum->message, sizeof sum->message, "Residual and Jacobian evaluation failed."); break;
        case LM_GRADIENT_TOL: snprintf(sum->message, sizeof sum->message, "Gradient tolerance reached."); break;
        case LM_MAX_TIME: snprintf(sum->message, sizeof sum->message, "Maximum solver time reached."); break;
        case LM_MAX_ITER: snprintf(sum->message, sizeof sum->message, "Maximum number of iterations reached."); break;
        case LM_MIN_RADIUS: snprintf(sum->message, sizeof sum->message, "Minimum trust region radius reached."); break;
        case LM_INVALID_STEPS: snprintf(sum->message, sizeof sum->message, "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps: %d", opt.max_num_consecutive_invalid_steps); break;
        case LM_PARAMETER_TOL: snprintf(sum->message, sizeof sum->message, "Parameter tolerance reached. Relative step_norm: %e <= %e.", hs->msg_a, hs->msg_b); break;
        case LM_FUNCTION_TOL: snprintf(sum->message, sizeof sum->message, "Function tolerance reached. |cost_change|/cost: %e <= %e", hs->msg_a, hs->msg_b); break;
        default: break;
    }
    sum->total_time_s = elapsed();
    sum->kernel_launches = ctx->launches - launches0;
    return SFMB200_OK;
}

int sfmb200_ba_solve(sfmb200_ctx* ctx, const sfmb200_ba_options* opt, int nc, int np, int nobs, double* cams6, double* pts3, double* focal,
                     const float* obs_xy, const int32_t* obs_cam, const int32_t* pt_off, sfmb200_ba_summary* summary) {
    if (!ctx || !focal || !summary) return SFMB200_ERR_INVALID;
    sfmb200_ba_problem* P = nullptr;
    int rc = sfmb200_ba_problem_create(ctx, nc, np, nobs, cams6, pts3, *focal, obs_xy, obs_cam, pt_off, &P);
    if (rc) return rc;
    if (ctx->nranks > 1) {            // peer-memory exchange instead of the NCCL all-reduce (collective: every rank is in this call)
        {
            std::lock_guard<std::mutex> lk(ctx->mu);
            rc = ba_auto_attach(P);
        }
        if (rc) { sfmb200_ba_problem_destroy(P); return rc; }
    }
    rc = sfmb200_ba_problem_run(P, opt, summary);
    if (!rc) rc = sfmb200_ba_problem_download(P, cams6, pts3, focal);
    sfmb200_ba_problem_destroy(P);
    return rc;
}

// ---- pose <-> parameter conversions of adjustBundle -------------------------------------------------------------
// ceres::RotationMatrixToAngleAxis<float>(R.t().val, aa) (:126): float arithmetic through a quaternion.
void sfmb200_rotmat_to_angle_axis_f32(const float* R, float* aa) {
    // R row-major; element (i,j) = R[3*i+j]
    const float trace = R[0] + R[4] + R[8];
    float q[4];
    if (trace >= 0.0f) {
        float t = sqrtf(trace + 1.0f);
        q[0] = 0.5f * t; t = 0.5f / t;
        q[1] = (R[7] - R[5]) * t; q[2] = (R[2] - R[6]) * t; q[3] = (R[3] - R[1]) * t;
    } else {
        int i = 0;
        if (R[4] > R[0]) i = 1;
        if (R[8] > R[4 * i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        float t = sqrtf(R[4 * i] - R[4 * j] - R[4 * k] + 1.0f);
        q[i + 1] = 0.5f * t; t = 0.5f / t;
        q[0] = (R[3 * k + j] - R[3 * j + k]) * t; q[j + 1] = (R[3 * j + i] + R[3 * i + j]) * t; q[k + 1] = (R[3 * k + i] + R[3 * i + k]) * t;
    }
    const float s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    if (s2 > 0.0f) {
        const float s = sqrtf(s2), c = q[0];
        const float two_theta = 2.0f * (c < 0.0f ? atan2f(-s, -c) : atan2f(s, c));
        const float kk = two_theta / s;
        aa[0] = q[1] * kk; aa[1] = q[2] * kk; aa[2] = q[3] * kk;
    } else { aa[0] = q[1] * 2.0f; aa[1] = q[2] * 2.0f; aa[2] = q[3] * 2.0f; }
}

// ceres::AngleAxisToRotationMatrix followed by the reference's transposing write-back (:203-209): row-major R.
void sfmb200_angle_axis_to_rotmat(const double* aa, double* R) {
    CamDerived d; const double cam[6] = {aa[0], aa[1], aa[2], 0, 0, 0};
    cam_derive(cam, d);
    for (int i = 0; i < 9; ++i) R[i] = d.R[i];
}

}  // extern "C"
