/*
 * sfmb200.h -- C ABI of the H100-native SfM hot path (libsfmb200.so).
 *
 * Drop-in boundary for the three compute stages of royshil/SfM-Toy-Library (SURVEY.md section 8b).
 * Plain pointers and sizes only; the caller owns every host buffer, the library owns device scratch
 * inside the context.  All entry points return 0 (SFMB200_OK) or an error code; sfmb200_last_error()
 * gives the text.  Unless a name ends in `_device`, pointers are HOST pointers and the call performs
 * the host<->device copies itself (this is the path the reference-side shim binds, INTEGRATION.md).
 *
 * Reference interfaces replaced (file:line relative to the reference repo):
 *   sfmb200_match_*        <- SfM2DFeatureUtilities::matchFeatures      SfMToyLib/SfM2DFeatureUtilities.h:44-46, .cpp:53-71
 *   sfmb200_triangulate*   <- SfMStereoUtilities::triangulateViews      SfMToyLib/SfMStereoUtilities.h:82-91,  .cpp:120-206
 *                             (+ GetAlignedPointsFromMatch gather)      SfMToyLib/SfMCommon.cpp:63-87
 *   sfmb200_ba_*           <- SfMBundleAdjustmentUtils::adjustBundle    SfMToyLib/SfMBundleAdjustmentUtils.h:44-49, .cpp:99-222
 *                             (+ SimpleReprojectionError)               SfMToyLib/SfMBundleAdjustmentUtils.cpp:58-97
 */
#ifndef SFMB200_H
#define SFMB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SFMB200_VERSION 100

enum {
    SFMB200_OK = 0,
    SFMB200_ERR_INVALID = 1,   /* bad argument / malformed problem                          */
    SFMB200_ERR_CUDA = 2,      /* CUDA runtime error (no device, launch failure, ...)       */
    SFMB200_ERR_NOMEM = 3,     /* device or host allocation failed                          */
    SFMB200_ERR_COMM = 4,      /* NCCL / multi-GPU error                                    */
    SFMB200_ERR_UNSUPPORTED = 5
};

typedef struct sfmb200_ctx sfmb200_ctx;

/* ---- context: one per GPU (one process per GPU in multi-GPU runs) --------------------------------------- */
int sfmb200_version(void);
int sfmb200_create(int device, sfmb200_ctx** ctx);          /* fails loudly (ERR_CUDA) when there is no GPU */
void sfmb200_destroy(sfmb200_ctx* ctx);
const char* sfmb200_last_error(const sfmb200_ctx* ctx);     /* ctx may be NULL: error of the last failed create */
void* sfmb200_stream(sfmb200_ctx* ctx);                     /* the cudaStream_t every kernel of this ctx runs on */
int sfmb200_synchronize(sfmb200_ctx* ctx);
int64_t sfmb200_kernel_launches(const sfmb200_ctx* ctx);    /* number of kernels this ctx has launched so far */

/* ---- a-1: descriptor matching --------------------------------------------------------------------------- */
/*
 * matchFeatures (SfM2DFeatureUtilities.cpp:53-71): for every query row the 2 nearest train rows by Hamming
 * distance (ties -> lower train index), keep the best iff (double)d0 < ratio * (double)d1, ascending queryIdx.
 * Pass ratio = (double)0.8f to reproduce NN_MATCH_RATIO (SfM2DFeatureUtilities.cpp:35).
 * q [nq*desc_bytes], t [nt*desc_bytes] row-major PACKED bytes (ORB: desc_bytes = 32); 1 <= desc_bytes <= 128.  The kernels are
 * instantiated for 16/32/64/128 bytes; any other width is zero-padded to the next one (every distance unchanged).
 * 32-byte descriptors run on the wgmma tensor-core kernel, the other widths on the XOR/POPC kernel.
 * out_q/out_t/out_d must hold nq entries; *out_n receives the number of survivors (imgIdx is always 0).
 * nt < 2 (undefined behaviour in the reference) yields *out_n = 0.
 * The reference calls this once per image pair with the same images again and again (SfM.cpp:166-206): uploaded images
 * stay resident in a context-owned arena keyed by (host pointer, rows, width, 64-bit content hash), so a repeated image costs
 * neither an upload nor an expansion.  SFMB200_MATCH_CACHE=0 disables the arena.  Safe to call from several host threads.
 */
int sfmb200_match_knn2_ratio(sfmb200_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int desc_bytes,
                             double ratio, int32_t* out_q, int32_t* out_t, float* out_d, int* out_n);

/* L2 variant (cv::BFMatcher(NORM_L2), BASELINE.json configs[3] wording "SIFT-128"; the legacy tree's own L2 knn + ratio test is
 * legacy/SfMToyLib_Old/GPUSURFFeatureMatcher.cpp:100-124): float descriptors [n*dim], distance = sqrtf(sum of squared
 * differences).  Integer-valued descriptors in [0, 255] with dim <= 128 (what cv::SIFT produces) are matched EXACTLY as a
 * u8 x u8 -> s32 GEMM on the wgmma tensor cores (|a-b|^2 = |a|^2 + |b|^2 - 2<a,b>, every term an exact integer < 2^24, so the
 * float32 sum cv::batchDistance forms is reproduced bit for bit); anything else runs the fp32 SIMT kernel. */
int sfmb200_match_knn2_ratio_l2(sfmb200_ctx* ctx, const float* q, int nq, const float* t, int nt, int dim,
                                double ratio, int32_t* out_q, int32_t* out_t, float* out_d, int* out_n);

/* Batched all-pairs form of SfM::createFeatureMatchMatrix (SfM.cpp:157-212): descriptors of all images live in
 * HBM once; any list of (left,right) image pairs is matched in one launch sequence. */
typedef struct sfmb200_descset sfmb200_descset;
int sfmb200_descset_create(sfmb200_ctx* ctx, const uint8_t* desc /* concatenated rows */, const int32_t* img_off /* [n_img+1] row offsets */,
                           int n_img, int desc_bytes, sfmb200_descset** set);
/* same for L2 matching: float descriptors [rows*dim], dim <= 128, values must be integers in [0, 255] (SFMB200_ERR_UNSUPPORTED
 * otherwise).  sfmb200_match_pairs / _device then return float distances sqrtf(|a-b|^2) like cv::BFMatcher(NORM_L2). */
int sfmb200_descset_create_l2(sfmb200_ctx* ctx, const float* desc, const int32_t* img_off, int n_img, int dim, sfmb200_descset** set);
/* Destroy a set BEFORE its context.  One set at a time borrows its device memory from the context (no cudaMalloc / cudaFree per set,
 * the usual case: one set per run); further sets that are alive at the same time allocate their own. */
void sfmb200_descset_destroy(sfmb200_descset* set);
/* pairs [2*n_pairs] = (left,right) image ids.  Results of pair p are written to out_*[out_off[p] .. out_off[p]+out_cnt[p])
 * where out_off[p] = sum of the LEFT image sizes of pairs < p (computed here, returned in out_off [n_pairs+1]);
 * out_q/out_t/out_d must hold out_off[n_pairs] entries (<= n_pairs * max image size). */
int sfmb200_match_pairs(sfmb200_ctx* ctx, const sfmb200_descset* set, const int32_t* pairs, int n_pairs, double ratio,
                        int32_t* out_q, int32_t* out_t, float* out_d, int64_t* out_off, int32_t* out_cnt);
/* same, results stay on the device (the benchmark's resident-input timing): d_* are DEVICE pointers, pairs is host.
 * Survivors of all pairs are written DENSELY (pair-major, ascending queryIdx) to d_out_*[0 .. *d_total);
 * d_pair_start [n_pairs] = dense position of each pair's first survivor (0 for a pair without query rows).  Nothing is
 * synchronised.  n_pairs == 0 or no query rows at all: *d_total = 0.  *d_total = -1 reports a tensor-core pipeline failure
 * (an MMA completion barrier timed out) -- the outputs are then undefined. */
int sfmb200_match_pairs_device(sfmb200_ctx* ctx, const sfmb200_descset* set, const int32_t* pairs, int n_pairs, double ratio,
                               int32_t* d_out_q, int32_t* d_out_t, float* d_out_d, int32_t* d_pair_start, int64_t* d_total);

/* ---- image-pair batches: the input layout of the *_pairs calls ------------------------------------------------ */
/*
 * sfmb200_triangulate_pairs, sfmb200_find_camera_matrices_pairs and sfmb200_find_homography_pairs run a stage for many image pairs
 * in one call.  They take the same arrays, so one set of arrays serves all three:
 *   pts [img_off[n_img] * 2]   float pixel coordinates of the key points of all images; image i owns pts[2 img_off[i] .. 2 img_off[i+1])
 *   img_off [n_img + 1]        img_off[0] = 0, monotone
 *   pairs [n_pairs * 2]        (left image, right image), each in [0, n_img)
 *   match_q / match_t          per match, the key point index in the left / right image of its pair; pair p owns matches
 *                              match_off[p] .. match_off[p+1]
 *   match_off [n_pairs + 1]    match_off[0] = 0, monotone; M = match_off[n_pairs] matches in all
 * The arrays are checked on the host before any launch.  Each of the following gives SFMB200_ERR_INVALID with a message, and the
 * context stays usable: a needed array is NULL; img_off[0] != 0 or img_off not monotone; match_off[0] != 0 or match_off not
 * monotone; a pair names an image outside [0, n_img); M is above the call's limit; a match indexes outside its image's key points.
 * Where the three calls differ:
 *   - the limit on M: INT32_MAX for sfmb200_triangulate_pairs, INT32_MAX / 2 for the other two;
 *   - n_pairs == 0: sfmb200_triangulate_pairs and sfmb200_find_camera_matrices_pairs return SFMB200_OK without reading the arrays
 *     (after their option and K checks, where they have them); sfmb200_find_homography_pairs still checks img_off and pts.
 */

/* ---- a-2 (+ a-6): two-view triangulation ---------------------------------------------------------------- */
/*
 * triangulateViews (SfMStereoUtilities.cpp:120-206) on flat arrays:
 *   K [9] row-major float intrinsics; Pleft/Pright [12] row-major float 3x4 poses;
 *   pts_left [n_left*2], pts_right [n_right*2] float pixel coordinates (Features::points);
 *   match_q/match_t [m] indices into pts_left/pts_right (DMatch queryIdx/trainIdx); NULL,NULL = identity alignment
 *   (GetAlignedMatching, SfMCommon.cpp:120-126) with m <= min(n_left, n_right);
 *   max_reproj_px = MIN_REPROJECTION_ERROR = 10 (SfMStereoUtilities.cpp:42).
 * Outputs: X [m*3] float for every match, keep [m] (1 = passes the filter at :186-187), *n_keep.
 * The reference appends the kept points in match order with back references match_q[i]/match_t[i] (:192-202).
 */
int sfmb200_triangulate(sfmb200_ctx* ctx, const float* K, const float* Pleft, const float* Pright,
                        const float* pts_left, int n_left, const float* pts_right, int n_right,
                        const int32_t* match_q, const int32_t* match_t, int m, float max_reproj_px,
                        float* X, uint8_t* keep, int* n_keep);
/* device-resident variant: every array pointer is a DEVICE pointer (K, Pleft, Pright stay host). d_n_keep [1] int32. */
int sfmb200_triangulate_device(sfmb200_ctx* ctx, const float* K, const float* Pleft, const float* Pright,
                               const float* d_pts_left, const float* d_pts_right,
                               const int32_t* d_match_q, const int32_t* d_match_t, int m, float max_reproj_px,
                               float* d_X, uint8_t* d_keep, int32_t* d_n_keep);
/*
 * sfmb200_triangulate for every pair of an image-pair batch in one call; pts / img_off / pairs / match_q / match_t / match_off,
 * their checks and n_pairs == 0 are described under "image-pair batches" above.  Pair p's slices of X and keep and n_keep[p] are
 * bitwise what sfmb200_triangulate returns for that pair's matches and poses, whatever else is in the batch and wherever the pair
 * stands in it.  A pair with no matches gets n_keep 0.
 *   K [9] float row-major, shared by all pairs; poses [n_pairs * 24]: pair p's Pleft [12] then Pright [12], row-major 3x4 float.
 *   max_reproj_px as in sfmb200_triangulate.
 *   X [match_off[n_pairs] * 3], keep [match_off[n_pairs]]; n_keep [n_pairs] survivors per pair, may be NULL.
 * One upload, one download and one host synchronisation per call, with one launch of sfmb200_triangulate's kernel per pair that
 * has matches.
 */
int sfmb200_triangulate_pairs(sfmb200_ctx* ctx, const float* K, const float* poses, const float* pts, const int32_t* img_off, int n_img,
                              const int32_t* pairs, int n_pairs, const int32_t* match_q, const int32_t* match_t, const int64_t* match_off,
                              float max_reproj_px, float* X, uint8_t* keep, int32_t* n_keep);

/* ---- a-3 / a-4: bundle adjustment ----------------------------------------------------------------------- */
/* Options = the Ceres options the reference sets (SfMBundleAdjustmentUtils.cpp:171-177) + the Ceres defaults it
 * leaves alone (SURVEY.md appendix A.3).  sfmb200_ba_default_options() fills in exactly those. */
typedef struct {
    int max_num_iterations;                 /* 500  (:174) */
    double max_solver_time_in_seconds;      /* 10   (:176); <= 0 disables the cap */
    double function_tolerance;              /* 1e-6  */
    double gradient_tolerance;              /* 1e-10 */
    double parameter_tolerance;             /* 1e-8  */
    double initial_trust_region_radius;     /* 1e4   */
    double max_trust_region_radius;         /* 1e16  */
    double min_trust_region_radius;         /* 1e-32 */
    double min_relative_decrease;           /* 1e-3  */
    double min_lm_diagonal;                 /* 1e-6  */
    double max_lm_diagonal;                 /* 1e32  */
    int jacobi_scaling;                     /* 1     */
    int max_num_consecutive_invalid_steps;  /* 5     */
    int verbose;                            /* 1: one line per LM iteration on stdout (minimizer_progress_to_stdout, :173) */
    int profile;                            /* 1: time the dominant kernel with CUDA events (summary.schur_ms_*) */
    int l2_flush_mb;                        /* > 0: write a scratch buffer of this many MB between LM iterations (benchmark hygiene) */
} sfmb200_ba_options;

enum { SFMB200_BA_CONVERGENCE = 0, SFMB200_BA_NO_CONVERGENCE = 1, SFMB200_BA_FAILURE = 2 };

typedef struct {
    int termination_type;                   /* SFMB200_BA_* ; the reference writes results back only on CONVERGENCE (:182-185) */
    int num_iterations;                     /* LM iterations after iteration 0 */
    int num_successful_steps, num_unsuccessful_steps;
    int num_jacobian_passes;                /* residual+Jacobian evaluation passes over all observations (incl. Schur reduction) */
    int num_linear_solves;
    double initial_cost, final_cost;        /* 1/2 sum r^2 over ALL ranks' observations */
    double total_time_s;                    /* host wall clock of the LM loop */
    double schur_ms_total;                  /* profile=1: CUDA-event time of the point-elimination kernel (K3a), summed */
    int schur_launches;
    double pair_ms_total;                   /* profile=1: CUDA-event time of the camera-pair block kernel (K3c), summed */
    int pair_launches;
    double camera_ms_total;                 /* profile=1: CUDA-event time of the camera-major kernel (K3b), summed (one launch per schur launch) */
    double solve_ms_total;                  /* profile=1: CUDA-event time of the dense solve (K4: assemble, Cholesky, back substitution), summed */
    double flush_ms_total;                  /* profile=1 and l2_flush_mb > 0: CUDA-event time of the L2 flush writes, summed (not part of the algorithm) */
    int64_t kernel_launches;                /* kernels launched by this solve */
    char message[160];
} sfmb200_ba_summary;

void sfmb200_ba_default_options(sfmb200_ba_options* opt);

/* Host-only check of a flattened problem: CSR offsets monotone from 0 to nobs, cameras in [0, nc) and strictly ascending
 * inside a point (the std::map order of reference :146), at most 255 views per point.  sfmb200_ba_problem_create /
 * sfmb200_ba_solve run the same check; exported so that a host can validate without a device.  0 = valid; otherwise
 * SFMB200_ERR_INVALID / _UNSUPPORTED with the reason in `message`.
 * A problem this accepts is also accepted by sfmb200_ba_problem_create in the default (gather) Schur mode.  The atomics
 * ("red") Schur mode keeps a point's Schur terms in shared memory and supports at most 244 views per point: create refuses
 * more with SFMB200_ERR_UNSUPPORTED and "observations per point (k) exceed the shared-memory budget of the atomics ("red")
 * Schur mode".  That mode runs with SFMB200_BA_SCHUR=red, and create chooses it by itself for large problems whose pair
 * lists outgrow the gather mode's buffers: thousands of cameras, 2^31 - 1024 or more pairs of observations of one point summed
 * over the points, or per-camera-pair partial blocks beyond 256 MB. */
int sfmb200_ba_validate(int nc, int np, int nobs, const int32_t* obs_cam, const int32_t* pt_off, char* message, int message_len);

/*
 * Flattened adjustBundle problem (the layout the reference builds at :111-166):
 *   cams6 [nc*6]  angle-axis(3) + translation(3) per camera, world->camera (:123-134)
 *   pts3  [np*3]  3D points (:144)
 *   focal [1]     the single shared focal length (:138)
 *   obs_xy [nobs*2] float, principal point already subtracted in float (:149-153)
 *   obs_cam [nobs] camera index of each observation; pt_off [np+1] CSR: observations of point i are
 *   [pt_off[i], pt_off[i+1]), cameras strictly ascending within a point (std::map iteration order, :146).
 * In multi-GPU runs every rank passes ALL cameras and ITS OWN shard of points/observations; the reduced camera
 * system is summed over ranks (sfmb200_comm_*).  cams6/focal come back identical on every rank.
 */
typedef struct sfmb200_ba_problem sfmb200_ba_problem;
int sfmb200_ba_problem_create(sfmb200_ctx* ctx, int nc, int np, int nobs, const double* cams6, const double* pts3, double focal,
                              const float* obs_xy, const int32_t* obs_cam, const int32_t* pt_off, sfmb200_ba_problem** prob);
void sfmb200_ba_problem_destroy(sfmb200_ba_problem* prob);
int sfmb200_ba_problem_reset(sfmb200_ba_problem* prob);      /* parameters := the values given at create (device copy) */
int sfmb200_ba_problem_run(sfmb200_ba_problem* prob, const sfmb200_ba_options* opt, sfmb200_ba_summary* summary);
int sfmb200_ba_problem_download(sfmb200_ba_problem* prob, double* cams6, double* pts3, double* focal);
/* test/diagnostic hook: reduced camera(+focal) system of DENSE_SCHUR at the current parameters for a trust-region
 * radius: S [(6nc+1)^2] row-major symmetric, rhs [6nc+1], grad_cf [6nc+1] (unscaled gradient wrt cameras+focal),
 * cost.  Any output may be NULL.  Multi-GPU: summed over ranks. */
int sfmb200_ba_problem_reduced_system(sfmb200_ba_problem* prob, const sfmb200_ba_options* opt, double radius,
                                      double* S, double* rhs, double* grad_cf, double* cost);
/* The dense solve of the reduced system keeps its right-hand side (n = 6 nc + 1 doubles, padded to a multiple of 32 plus one) in
 * the shared memory of one CTA above 469 cameras.  On an H100 (227 KB per block) that allows n <= 29055, i.e. at most 4842
 * cameras; sfmb200_ba_problem_create refuses larger problems with SFMB200_ERR_UNSUPPORTED and says so in the message. */
/* test/diagnostic hook: the dense solve of sfmb200_ba_problem_run (chol.cuh) on `count` SPD systems, back to back on ONE set of
 * buffers (solve number + 1 per system, as in the LM loop).  A [count][n][n] row-major, only the lower triangle read;
 * b [count][n].  grid: CTAs of the factorisation, 0 = what a BA problem of this n uses, otherwise 1 .. co-resident count
 * (larger is refused: deadlock freedom rests on it).  backsolve: 0 = a BA problem's choice, 1 = cluster (refused where its
 * slices do not fit), 2 = one CTA.  x [count][n]; L [count][n][n] lower factor or NULL; fail [count] the raw failure counter:
 * 0 = every pivot and paired 2x2 minor was a normal positive double, >= 1000 = a wait timed out.  Any n >= 1. */
int sfmb200_dense_spd_solve(sfmb200_ctx* ctx, int n, int count, const double* A, const double* b, int grid, int backsolve,
                            double* x, double* L, int32_t* fail);

/* Multi-GPU exchange over PEER MEMORY instead of NCCL: every rank exports the CUDA-IPC handle of its problem's exchange
 * buffer, the host all-gathers the handles (rank order) and every rank attaches them.  From then on the reduced camera
 * system is summed by kernels that load the peers' partial buffers directly over NVLink.  Needs sfmb200_comm_init
 * (rank / size) first; all ranks must create their problems before anyone attaches. */
#define SFMB200_IPC_HANDLE_BYTES 64
int sfmb200_ba_problem_ipc_handle(sfmb200_ba_problem* prob, uint8_t* handle /* [SFMB200_IPC_HANDLE_BYTES] */);
int sfmb200_ba_problem_ipc_attach(sfmb200_ba_problem* prob, const uint8_t* handles /* [nranks * SFMB200_IPC_HANDLE_BYTES] */);

/* one-shot: create + run + download + destroy (what the adjustBundle shim calls). cams6/pts3/focal are updated in
 * place with the final iterate whatever the termination type; the CONVERGENCE-only write-back rule is the caller's. */
int sfmb200_ba_solve(sfmb200_ctx* ctx, const sfmb200_ba_options* opt, int nc, int np, int nobs,
                     double* cams6, double* pts3, double* focal,
                     const float* obs_xy, const int32_t* obs_cam, const int32_t* pt_off, sfmb200_ba_summary* summary);

/* pose <-> parameter conversions of adjustBundle (:115-135 in float, :192-215 in double), exposed so the shim and
 * the tests share them: R row-major 3x3. */
void sfmb200_rotmat_to_angle_axis_f32(const float* R_rowmajor, float* angle_axis);
void sfmb200_angle_axis_to_rotmat(const double* angle_axis, double* R_rowmajor);

/* ---- f-2 ("next" row of SURVEY.md 8): batched RANSAC hypothesis scoring ----------------------------------- */
/*
 * The three RANSAC stages on either side of triangulation in the reference driver:
 *   findHomographyInliers        SfMStereoUtilities.cpp:51-72   cv::findHomography(RANSAC, RANSAC_THRESHOLD = 10 px) -> countNonZero(mask)
 *   findCameraMatricesFromMatch  SfMStereoUtilities.cpp:74-118  cv::findEssentialMat(focal, pp, RANSAC, 0.999, 1.0) -> mask prunes the matches
 *   findCameraPoseFrom2D3DMatch  SfMStereoUtilities.cpp:208-243 cv::solvePnPRansac(100 iterations, 10 px, 0.99) -> inlier ratio test
 * OpenCV scores one hypothesis at a time; this scores ALL `nh` hypotheses of a run against all `n` correspondences in one launch
 * sequence, with OpenCV's error formulas and arithmetic types (float transfer error for H, double Sampson error for E, squared
 * float reprojection error for a pose) and its inlier rule  err <= (float)(threshold^2).  Hypotheses are generated on the host.
 *   model      SFMB200_MODEL_HOMOGRAPHY: a = left points [n*2], b = right points [n*2], hyp [nh*9] row-major H (any scale; normalised to h22 = 1)
 *              SFMB200_MODEL_ESSENTIAL:  a, b as above (PIXELS), hyp [nh*9] E, aux9 = {focal, cx, cy, ...}: points are normalised
 *                                        (x - cx)/focal in double like cv::findEssentialMat(points, focal, pp); pass threshold / focal
 *              SFMB200_MODEL_POSE:       a = 3D points [n*3], b = image points [n*2], hyp [nh*12] row-major [R|t], aux9 = K (row-major 3x3)
 *   outputs    inlier_counts [nh] (may be NULL); *best_index = hypothesis with the most inliers (ties -> lowest index, the one
 *              OpenCV's sequential loop would have kept), -1 when nh == 0; best_mask [n] (may be NULL) = its inlier mask.
 */
enum { SFMB200_MODEL_HOMOGRAPHY = 0, SFMB200_MODEL_ESSENTIAL = 1, SFMB200_MODEL_POSE = 2 };
int sfmb200_ransac_score(sfmb200_ctx* ctx, int model, const float* a, const float* b, int n, const double* hyp, int nh, const double* aux9,
                         double threshold, int32_t* inlier_counts, int32_t* best_index, uint8_t* best_mask);

/* ---- f-2: essential-matrix RANSAC and pose recovery, all on the device ----------------------------------------- */
/*
 * findCameraMatricesFromMatch (SfMStereoUtilities.cpp:74-118):
 *     E = findEssentialMat(left, right, focal, pp, RANSAC, 0.999, 1.0, mask);  recoverPose(E, left, right, R, t, focal, pp, mask);
 * in one call.  Points are normalised x = ((double)px - cx) / focal with focal = K[0], (cx, cy) = (K[2], K[5]); the threshold
 * becomes threshold_px / focal.  max_iters samples of 5 distinct correspondences are drawn by the sampler the options name,
 * every sample is solved by the five-point solver (up to 10 E, real roots in ascending order), every solution is scored with the
 * Sampson error and inlier rule of sfmb200_ransac_score, and OpenCV's sequential loop (RANSACPointSetRegistrator::run) is replayed
 * over the counts in (sample, solution) order: a solution replaces the best one only if its count exceeds max(best count, 4),
 * every improvement recomputes the sample budget with RANSACUpdateNumIters(confidence, outlier ratio, 5, budget), and the loop
 * stops at the budget.
 *   SFMB200_SAMPLER_SEEDED (default): a counter-based generator (splitmix64 keyed by seed, sample and draw; a repeated index is
 *   redrawn).  cv:: draws its samples from its own RNG, so the result agrees with cv::findEssentialMat only statistically.
 *   SFMB200_SAMPLER_OPENCV: cv::findEssentialMat's own samples; seed is ignored.  Checked against cv2 4.13:
 *     identical: the samples and their order (cv::RNG restarted at (uint64)-1 for every pair, getSubset's redraws of a repeated
 *     index, no subset check), the per-solution inlier counts as far as the solutions agree, the selection and `iterations`;
 *     equal to rounding: E, about 1e-12 after sign and scale normalisation on the crazyhorse pairs (up to a few 1e-7 where the
 *     winning sample is ill-conditioned); hence inlier_mask, R, t and pose_mask;
 *     could in principle differ: a point whose Sampson error lies within rounding of the threshold; a sample on which the two
 *     five-point solvers disagree (ill-conditioned), if it would hold the winner; and a tie between two solutions of one sample
 *     that both improve on the best and decide the final winner: here the solution with the smaller root z wins (ascending
 *     order), in cv:: the one its polynomial solver lists first.  None of these changes a result on the crazyhorse pairs.
 * The pose is recoverPose's: E = U diag(s, s, 0) V^T, candidates [U W V^T | t], [U W^T V^T | t], [.. | -t], [.. | -t]
 * with t = U[:, 2]; a point counts for a candidate when its DLT triangulation against [I|0] has Q2 Q3 > 0, depth < distance_thresh in
 * the first camera, depth in (0, distance_thresh) in the second and its RANSAC inlier flag set; the first candidate whose count is
 * >= all others wins.
 *   K [9] float row-major; points / match_q / match_t as in sfmb200_triangulate (NULL, NULL = aligned).
 *   E [9], R [9], t [3] double (unit-norm t); any may be NULL.  inlier_mask [m] = findEssentialMat's mask, pose_mask [m] =
 *   recoverPose's (the pruning mask); either may be NULL.  opt NULL = defaults.  summary may be NULL.
 *   m < 5 or no model: SFMB200_OK with summary.found = 0, E / R / t / masks zero.
 *   m == 5: cv::findEssentialMat returns every solution of the one sample stacked (and the reference's recoverPose would then
 *   fail on the 3n x 3 matrix); here the one sample goes through the same selection as every other call.  Under
 *   SFMB200_SAMPLER_OPENCV that sample is the five points in their order, as cv:: solves them.
 *   SFMB200_ERR_INVALID: bad options (including a sampler other than the two below), a NULL K, a zero or non-finite focal length.
 * Same options, same inputs: bitwise-identical outputs.  One host synchronisation per call.
 */
enum { SFMB200_SAMPLER_SEEDED = 0, SFMB200_SAMPLER_OPENCV = 1 };
typedef struct {
    int max_iters;            /* 1000  cv::findEssentialMat default; >= 1 */
    double confidence;        /* 0.999 (SfMStereoUtilities.cpp:97); in (0, 1) */
    double threshold_px;      /* 1.0   (:97); > 0 */
    double distance_thresh;   /* 50    cv::recoverPose default; > 0 */
    uint64_t seed;            /* 0     SFMB200_SAMPLER_SEEDED only */
    int sampler;              /* SFMB200_SAMPLER_SEEDED; or SFMB200_SAMPLER_OPENCV */
} sfmb200_essential_options;
typedef struct {
    int found;                /* 1: a model with more than 4 inliers */
    int n_inliers;            /* inliers of E (findEssentialMat's mask) */
    int n_good;               /* points that pass the cheirality test (recoverPose's return value) */
    int iterations;           /* samples the sequential loop visited */
    int n_samples;            /* samples drawn and solved */
    int n_hypotheses;         /* solutions of all samples */
} sfmb200_essential_summary;
void sfmb200_essential_default_options(sfmb200_essential_options* opt);
int sfmb200_find_camera_matrices(sfmb200_ctx* ctx, const float* K, const float* pts_left, int n_left, const float* pts_right, int n_right,
                                 const int32_t* match_q, const int32_t* match_t, int m, const sfmb200_essential_options* opt,
                                 double* E, double* R, double* t, uint8_t* inlier_mask, uint8_t* pose_mask, sfmb200_essential_summary* summary);
/* Test hooks.  sfmb200_five_point: the device five-point solver on ns given samples, x1 / x2 [ns][5][2] normalised coordinates ->
 * E [ns][10][9] (unit Frobenius norm, real roots in ascending order), nsol [ns].
 * sfmb200_essential_last_trace: the last sfmb200_find_camera_matrices call's samples [cap][5], solution counts nsol [cap] and
 * per-solution inlier counts [cap * 10] in (sample, solution) order, for its first min(cap, n_samples) samples; any output may
 * be NULL.  Returns that call's n_samples (0 before any call), or -1 on bad arguments.  After a
 * sfmb200_find_camera_matrices_pairs call it describes that call's pair if it had exactly one, and returns 0 otherwise. */
int sfmb200_five_point(sfmb200_ctx* ctx, const double* x1, const double* x2, int ns, double* E, int32_t* nsol);
int sfmb200_essential_last_trace(sfmb200_ctx* ctx, int cap, int32_t* samples, int32_t* nsol, int32_t* counts);
/*
 * sfmb200_find_camera_matrices for every pair of an image-pair batch in one call; pts / img_off / pairs / match_q / match_t /
 * match_off, their checks and n_pairs == 0 are described under "image-pair batches" above.  Pair p's outputs
 * (E, R, t, its slices of both masks, summary[p]) are bitwise what sfmb200_find_camera_matrices returns for that pair's matches
 * with the same options, whatever else is in the batch and wherever the pair stands in it: one seed covers the call and every
 * pair draws its samples from it as a single call does (under SFMB200_SAMPLER_OPENCV from its own cv::RNG((uint64)-1)).  Per pair as in the single call: m < 5 gives found = 0 and zeros, m == 5
 * one sample, no model found = 0 with zeros.
 *   K [9] float row-major, shared by all pairs.
 *   E [n_pairs * 9], R [n_pairs * 9], t [n_pairs * 3]: any may be NULL.  inlier_mask / pose_mask [match_off[n_pairs]]: either
 *   may be NULL.  summary [n_pairs]: may be NULL.  opt NULL = defaults.
 * The option and K checks of the single call come before the batch's.  One upload, one download, one host synchronisation per
 * call.  The pairs run in
 * consecutive groups whose hypotheses (10 x 96 B per sample, 0.96 MB per pair at max_iters 1000) fit 256 MB of device memory,
 * enqueued back to back.
 */
int sfmb200_find_camera_matrices_pairs(sfmb200_ctx* ctx, const float* K, const float* pts, const int32_t* img_off, int n_img,
                                       const int32_t* pairs, int n_pairs, const int32_t* match_q, const int32_t* match_t,
                                       const int64_t* match_off, const sfmb200_essential_options* opt, double* E, double* R, double* t,
                                       uint8_t* inlier_mask, uint8_t* pose_mask, sfmb200_essential_summary* summary);

/* ---- f-2: camera pose from 2D-3D matches (PnP RANSAC + refit), all on the device ------------------------------ */
/*
 * findCameraPoseFrom2D3DMatch (SfMStereoUtilities.cpp:208-243):
 *     solvePnPRansac(points3D, points2D, K, distortion, rvec, t, false, 100, RANSAC_THRESHOLD = 10, 0.99, inliers)
 * in one call.  max_iters samples of 5 distinct correspondences are drawn from the generator of the essential-matrix RANSAC
 * (splitmix64 keyed by seed, sample and draw; a repeated index is redrawn).  Every sample is solved by EPnP in fp64 (at most one
 * pose; a degenerate sample -- coincident, collinear or coplanar 3D points, a rank-deficient system, a non-finite result -- gives
 * none).  Every pose is scored with the reprojection error and inlier rule of sfmb200_ransac_score (SFMB200_MODEL_POSE: double
 * projection, float difference, err <= (float)(threshold_px^2)), and OpenCV's sequential loop (RANSACPointSetRegistrator::run with
 * model_points = 5) is replayed over the counts in sample order: a pose replaces the best one only if its count exceeds
 * max(best count, 4), every improvement recomputes the sample budget with RANSACUpdateNumIters(confidence, outlier ratio, 5,
 * budget), and the loop stops at the budget.  cv:: draws its samples from its own RNG, so the RANSAC agrees with cv:: only
 * statistically.
 * Refit: with 6 or more inliers, damped Gauss-Newton (Levenberg-Marquardt) on (angle-axis, t) from the winner's pose minimises the
 * summed squared pixel reprojection error over the winner's inliers, at most refine_iters iterations, stopping when the relative
 * step or cost change falls below 1e-10: the least-squares minimum cv::solvePnP(SOLVEPNP_ITERATIVE) reaches on the same inliers.
 * If the refit does not lower the cost, the RANSAC pose is returned with summary.refined = 0.
 *   K [9] float row-major: fx = K[0], fy = K[4], cx = K[2], cy = K[5]; no distortion.  pts3 [m*3], pts2 [m*2] float.
 *   rvec [3] angle-axis, R [9] row-major (R = Rodrigues(rvec)), t [3], double; inlier_mask [m] = the RANSAC winner's inliers
 *   (solvePnPRansac's `inliers` output, before the refit; summary.n_inliers is their number).  Any output may be NULL.  opt NULL
 *   = defaults.  A correspondence with a non-finite coordinate is never an inlier.
 *   m < 5: SFMB200_OK with summary.found = 0 and zero outputs (cv::solvePnPRansac runs P3P at m == 4 and asserts below that).
 *   m == 5: EPnP on the five points, mask all ones, no refit (solvePnPRansac's model_points == npoints branch); found = 0 when
 *   the five points are degenerate.
 *   No pose with more than 4 inliers: found = 0 and zero outputs.
 *   SFMB200_ERR_INVALID: bad options, a NULL K, NULL points with m > 0, m < 0, a non-finite K entry, fx <= 0 or fy <= 0.
 * Four launches (solve, score, select, mask + refit), one upload, one download, one host synchronisation per call.  Same seed,
 * same inputs: bitwise-identical outputs.
 */
typedef struct {
    int max_iters;            /* 100   (SfMStereoUtilities.cpp:225); in [1, 2^24] */
    double confidence;        /* 0.99  (:225); in (0, 1) */
    double threshold_px;      /* 10    RANSAC_THRESHOLD (:41); finite, > 0 */
    int refine_iters;         /* 20    iterations of the refit; 0 = no refit (the RANSAC pose) */
    uint64_t seed;            /* 0 */
} sfmb200_pose_options;
typedef struct {
    int found;                /* 1: a pose with more than 4 inliers (m == 5: EPnP succeeded) */
    int n_inliers;            /* inliers of the RANSAC winner (the mask) */
    int iterations;           /* samples the sequential loop visited */
    int n_samples;            /* samples drawn and solved */
    int n_hypotheses;         /* samples that gave a pose */
    int refined;              /* 1: the returned pose is the refit's */
} sfmb200_pose_summary;
void sfmb200_pose_default_options(sfmb200_pose_options* opt);
int sfmb200_find_camera_pose(sfmb200_ctx* ctx, const float* K, const float* pts3, const float* pts2, int m, const sfmb200_pose_options* opt,
                             double* rvec, double* R, double* t, uint8_t* inlier_mask, sfmb200_pose_summary* summary);
/* Test hooks.  sfmb200_epnp: the device minimal solver on ns given samples, X [ns][5][3] world points, uv [ns][5][2] pixels, K [9]
 * double row-major -> Rt [ns][12] row-major [R|t] (zeros where ok = 0), ok [ns].  The RANSAC runs the same machine code.
 * sfmb200_pose_last_trace: the last sfmb200_find_camera_pose call's samples [cap][5] and per-sample inlier counts [cap] (-1: the
 * sample gave no pose), for its first min(cap, n_samples) samples; either output may be NULL.  Returns that call's n_samples (0
 * before any call or after a call with m < 5), or -1 on bad arguments. */
int sfmb200_epnp(sfmb200_ctx* ctx, const double* X, const double* uv, const double* K, int ns, double* Rt, uint8_t* ok);
int sfmb200_pose_last_trace(sfmb200_ctx* ctx, int cap, int32_t* samples, int32_t* counts);

/* ---- f-2: homography RANSAC for many image pairs, all on the device -------------------------------------------- */
/*
 * findHomographyInliers (SfMStereoUtilities.cpp:51-72) for every pair of a batch in one call:
 *     H = findHomography(left, right, RANSAC, threshold_px, mask, max_iters, confidence);  count = countNonZero(mask)
 * Identical to OpenCV 4.x (checked against cv2 4.13):
 *   - the samples: cv::RNG seeded with (uint64)-1 at the start of every pair, getSubset's redraws of repeated indices and of quads
 *     that fail the collinearity or orientation checks, so the same quads in the same order;
 *   - the inlier test (float transfer error with H cast to float, err <= (float)(threshold^2)), the selection (a model replaces
 *     the best only with more than max(best, 3) inliers) and RANSACUpdateNumIters(confidence, outlier ratio, 4, budget);
 *   - hence the RANSAC inlier set, ransac_inliers and iterations;
 *   - the returned mask and n_inliers: the inliers of the refined H, as cv::findHomography returns them.
 * Not bit-identical: H itself.  The 4-point and least-squares DLT (normalised, eigenvector of the smallest eigenvalue of L^T L by
 * cyclic Jacobi) and the Levenberg-Marquardt refinement (LMSolverImpl's schedule, 8 x 8 solves by Gaussian elimination) agree with
 * OpenCV's to rounding, about 1e-7 of max|H| at worst on the crazyhorse pairs.  A point whose error lies within that rounding of the
 * threshold could in principle flip; on those pairs the closest point is 1e-3 threshold^2 away.
 * n == 4 follows findHomography: the DLT of the four points, no checks, no refinement, mask all ones.  n < 4 or no model: found = 0,
 * n_inliers = 0, H and mask zero (the reference's `homography.empty()` branch).
 *   pts / img_off / pairs / match_q / match_t / match_off: an image-pair batch; the layout, its checks and n_pairs == 0 are
 *   described under "image-pair batches" above.  The option checks come first, and record_trace = 1 refuses n_pairs * max_iters
 *   above INT32_MAX / 4.
 *   H [n_pairs * 9]            row-major, h22 = 1; may be NULL.  mask [match_off[n_pairs]]: may be NULL.  summary [n_pairs]: may be NULL.
 * One CTA per pair, one host synchronisation per call.  Same inputs: bitwise-identical outputs, whether a pair is alone in a call or
 * batched with others.  There is no seed: reproducing OpenCV's sample sequence is the point.
 */
typedef struct {
    int max_iters;            /* 2000  cv::findHomography default; >= 1 */
    double confidence;        /* 0.995 cv::findHomography default; in (0, 1) */
    double threshold_px;      /* 10    RANSAC_THRESHOLD (SfMStereoUtilities.cpp:41); > 0 */
    int refine_iters;         /* 10    Levenberg-Marquardt iterations of cv::findHomography; >= 1 */
    int record_trace;         /* 0     1: keep every visited sample for sfmb200_homography_last_trace (20 bytes x max_iters per pair) */
} sfmb200_homography_options;
typedef struct {
    int found;                /* 1: a model (cv::findHomography returned a non-empty H) */
    int n_inliers;            /* countNonZero(mask): inliers of the refined H */
    int ransac_inliers;       /* inliers of the best RANSAC model, before the refinement */
    int iterations;           /* samples the sequential loop visited */
} sfmb200_homography_summary;
void sfmb200_homography_default_options(sfmb200_homography_options* opt);
int sfmb200_find_homography_pairs(sfmb200_ctx* ctx, const float* pts, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs,
                                  const int32_t* match_q, const int32_t* match_t, const int64_t* match_off,
                                  const sfmb200_homography_options* opt, double* H, uint8_t* mask, sfmb200_homography_summary* summary);
/* Test hook: the samples the last sfmb200_find_homography_pairs call with record_trace = 1 visited for pair `pair`, in order: quads
 * [cap][4] (indices into the pair's matches) and RANSAC inlier counts [cap] (-1: the DLT gave no model), the first min(cap, visited).
 * Either output may be NULL.  Returns the number visited, or -1 (bad arguments, or no trace recorded). */
int sfmb200_homography_last_trace(sfmb200_ctx* ctx, int pair, int cap, int32_t* quads, int32_t* counts);

/* ---- f-3 ("next" row of SURVEY.md 8): ORB feature extraction, the step before matching ------------------------ */
/*
 * SfM2DFeatureUtilities::extractFeatures (SfMToyLib/SfM2DFeatureUtilities.h:41-42, .cpp:46-51):
 *     mDetector = ORB::create(5000);                                                         (.cpp:39)
 *     mDetector->detectAndCompute(image, noArray(), features.keyPoints, features.descriptors);   (.cpp:48)
 * called once per image by SfM::extractFeatures (SfM.cpp:141-154) on the BGR images cv::imread returned (SfM.cpp:124).
 * ORB::create's other parameters are OpenCV's defaults (scaleFactor 1.2f, 8 levels, edgeThreshold 31, firstLevel 0, WTA_K 2,
 * HARRIS_SCORE, patchSize 31, fastThreshold 20).  Output is bit-identical to OpenCV's (cv2 4.13 in this image): the same key points
 * in the same order with the same pt / size / angle / response / octave, and the same 32-byte descriptors.
 *   image        8-bit pixels, channels = 1 (grey) or 3 (B,G,R interleaved; converted like cvtColor(COLOR_BGR2GRAY)); row_stride in
 *                bytes (0 = packed rows).  8 <= width, height <= 65535, width * height <= 2^28.  JPEG files decode with sfmb200_decode_jpeg_batch below.
 *   keypoints    [max_keypoints] records with the memory layout of cv::KeyPoint (28 bytes), so a shim can copy them straight into a
 *                std::vector<cv::KeyPoint>; class_id = -1.  KeyPointsToPoints (SfMCommon.cpp:89-94) is the x,y prefix of every record.
 *   descriptors  [max_keypoints * 32]
 *   n_keypoints  number of key points found.  OpenCV keeps ties at the selection thresholds, so this can exceed nfeatures; when it
 *                exceeds max_keypoints only the first max_keypoints records were written -- call again with a larger capacity.
 * The batch form extracts all images of a run (equal sizes) with shared launches and three host round trips per batch; keypoints /
 * descriptors / n_keypoints are then [n_images][max_keypoints] / [n_images][max_keypoints * 32] / [n_images].
 */
typedef struct sfmb200_keypoint { float x, y, size, angle, response; int32_t octave, class_id; } sfmb200_keypoint;
int sfmb200_orb_detect_and_compute(sfmb200_ctx* ctx, const uint8_t* image, int width, int height, int channels, size_t row_stride, int nfeatures,
                                   int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints);
int sfmb200_orb_detect_and_compute_batch(sfmb200_ctx* ctx, const uint8_t* const* images, int n_images, int width, int height, int channels,
                                         size_t row_stride, int nfeatures, int max_keypoints, sfmb200_keypoint* keypoints,
                                         uint8_t* descriptors, int32_t* n_keypoints);
/* Host-side pieces of the stage, exported so that they can be tested without a GPU: the pyramid layout (8 levels: size, scale, key point
 * quota), the tap table of resize(INTER_LINEAR_EXACT), and KeyPointsFilter::retainBest (returns the number of survivors, their
 * original indices in OpenCV's output order in `order`; -1 on bad arguments). */
int sfmb200_orb_layout(int width, int height, int nfeatures, int32_t* level_w, int32_t* level_h, float* level_scale, int32_t* level_quota);
int sfmb200_orb_linear_exact_taps(int src, int dst, int32_t* i0, int32_t* i1, int32_t* weight);
int sfmb200_orb_retain_best(const float* response, int n, int n_points, int32_t* order);
/* Inspection of the last extraction (parity tests): one level of image `image` of the last batch; stage 0 = pyramid, 1 = blurred
 * pyramid the descriptors sample, 2 = FAST score map.  out [level_w * level_h] with that image's own level size. */
int sfmb200_orb_download_level(sfmb200_ctx* ctx, int stage, int image, int level, uint8_t* out);
/* Host wall-clock (ms) of the phases of the last extraction call: 0 staging + upload + kernel enqueue, 1 wait for detection,
 * 2 candidate read-back, 3 first retainBest, 4 Harris round trip, 5 second retainBest, 6 describe round trip, 7 copy-out. */
int sfmb200_orb_last_timings(const sfmb200_ctx* ctx, double* ms8);
/* Self-test of the context's host thread pool (csrc/host_pool.h; staging and retainBest tasks of the ORB stage run on it): `rounds`
 * parallel loops of varying length on `n_threads` threads; returns a checksum >= 0, -1 on bad arguments, -2 on a wrong result. */
int64_t sfmb200_host_pool_selftest(int n_threads, int rounds, int max_tasks);

/* ---- f-3: JPEG decoding, the step before ORB extraction --------------------------------------------------------- */
/*
 * The imread loop of SfM::setImagesDirectory (SfM.cpp:123-135) for all images of a run in one call:  mImages.push_back(imread(file)).
 * The output is byte-identical to cv::imread(file, IMREAD_COLOR) with the libjpeg-turbo 3.1 OpenCV 4.13 bundles: ISLOW integer IDCT,
 * fancy upsampling, libjpeg's integer YCbCr -> RGB tables, B,G,R order, EXIF orientation (tag 0x0112 of IFD0 in the first APP1)
 * applied -- orientations 5-8 swap width and height.  A grey file gives three equal channels.
 * Supported: baseline and extended sequential Huffman JPEG (SOF0 / SOF1), 8-bit, 1 component or 3 (YCbCr) with the sampling
 * cv::imencode writes (4:4:4, 4:2:2, 4:2:0, 4:4:0, 4:1:1), optimised or standard Huffman tables, restart intervals, any size, any
 * APPn / COM segments.  Progressive, arithmetic-coded, lossless, 12-bit, 4-component and RGB (Adobe transform 0) files and other
 * sampling factors return SFMB200_ERR_UNSUPPORTED.  Truncated or corrupt data returns SFMB200_ERR_INVALID -- unlike libjpeg, which
 * warns, pads and returns an image.  sfmb200_last_error names the image and the reason; the context stays usable.
 *
 * sfmb200_jpeg_info: host only (no context, no GPU): the output size (after orientation) and the component count of the file, or the
 * status a decode would return.
 * sfmb200_decode_jpeg_batch: decodes the n files data[i] [size[i] bytes] into caller-owned host buffers out_bgr[i], rows of
 * out_stride[i] bytes (out_stride NULL or 0 = packed rows, width * 3).  The images may differ in size.  One upload of all
 * entropy-coded data, one download, one host synchronisation per call.  An image decodes to the same bytes alone or in a batch.  If
 * any file fails, the call returns that status and the outputs are unspecified.  At most 65535 files and 512 MB of entropy-coded data
 * per call.
 * sfmb200_jpeg_last_stats: the Huffman phase of the last call: [0] subsequences of 1024 bits, [1] codewords decoded by the first pass,
 * [2] codewords decoded again to synchronise, [3] parallel synchronisation rounds run, [4] subsequences the in-order sweep re-decoded,
 * [5] bytes uploaded, [6] bytes downloaded.
 */
int sfmb200_jpeg_info(const uint8_t* data, size_t size, int* width, int* height, int* components);
int sfmb200_decode_jpeg_batch(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, uint8_t* const* out_bgr,
                              const size_t* out_stride);
int sfmb200_jpeg_last_stats(const sfmb200_ctx* ctx, int64_t* stats7);

/* ---- f-3: image downscale, the optional step after imread -------------------------------------------------------- */
/*
 * The downscale of SfM::setImagesDirectory (SfM.cpp:127-129, main.cpp's -s/--downscale):
 *     if (mDownscaleFactor != 1.0) resize(img, img, Size(), mDownscaleFactor, mDownscaleFactor);
 * byte-identical to OpenCV 4.13's cv::resize with the default INTER_LINEAR on 8-bit B,G,R images.  `scale` is the reference's float
 * factor widened to double.  Output size cvRound(w * scale) x cvRound(h * scale) (half to even: 173 * 0.5 -> 86, 175 * 0.5 -> 88).
 * A factor of exactly 0.5 takes OpenCV's 2x2 area path; any other factor its Q11 fixed-point bilinear path; an image whose size does
 * not change is copied, and a factor of exactly 1 returns the input bytes (the reference does not call resize then).  A scale that is
 * not finite or <= 0, or that leaves an image with no pixels, returns SFMB200_ERR_INVALID (cv::resize asserts).
 *
 * sfmb200_resize_size: host only (no context, no GPU): the output size of a w x h image.
 * sfmb200_resize_batch: resizes the n host images src[i] (w[i] x h[i], B,G,R, rows of src_stride[i] bytes) into caller-owned host
 * buffers dst[i] sized with sfmb200_resize_size, rows of dst_stride[i] bytes (a stride array NULL or an entry 0 = packed rows).  The
 * images may differ in size.  One upload, one launch, one download and one host synchronisation per call; a factor of 1 copies on
 * the host.  At most 65535 images per call.
 * sfmb200_decode_jpeg_batch_scaled: sfmb200_decode_jpeg_batch followed by the downscale on the device, in one call: only the resized
 * images are downloaded (sfmb200_jpeg_last_stats [6] counts them).  Each out_bgr[i] holds the size sfmb200_resize_size gives for the
 * size sfmb200_jpeg_info reports; out_stride as in sfmb200_decode_jpeg_batch.  scale == 1 returns exactly the bytes of
 * sfmb200_decode_jpeg_batch.
 */
int sfmb200_resize_size(int w, int h, double scale, int* dw, int* dh);
int sfmb200_resize_batch(sfmb200_ctx* ctx, const uint8_t* const* src, const int* w, const int* h, const size_t* src_stride, int n,
                         double scale, uint8_t* const* dst, const size_t* dst_stride);
int sfmb200_decode_jpeg_batch_scaled(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale,
                                     uint8_t* const* out_bgr, const size_t* out_stride);

/* ---- f-3: JPEG files to ORB features in one call ----------------------------------------------------------------- */
/*
 * setImagesDirectory's imread (+ resize) loop and SfM::extractFeatures for all images of a run, with the images staying on the device
 * between the decode and ORB: per image the key points and descriptors of
 *     ORB::create(nfeatures)->detectAndCompute(resize(imread(file), Size(), scale, scale))      (no resize when scale == 1)
 * bit-identical to OpenCV, exactly what sfmb200_decode_jpeg_batch[_scaled] followed by sfmb200_orb_detect_and_compute gives.  The
 * images may differ in size (EXIF orientations 5-8 swap width and height); they share every launch.
 *   data, size, n, scale   as in sfmb200_decode_jpeg_batch_scaled; the same statuses for unsupported or corrupt files, detected before
 *                          any ORB work.  A decoded (resized) image with a side below 8 pixels returns SFMB200_ERR_INVALID, one over 2^28
 *                          pixels SFMB200_ERR_UNSUPPORTED, before any launch; the message names the image.
 *   keypoints, descriptors, n_keypoints   [n][max_keypoints] / [n][max_keypoints * 32] / [n], as in sfmb200_orb_detect_and_compute_batch
 *                          (n_keypoints may exceed max_keypoints: call again with a larger capacity).
 *   out_bgr, out_stride    NULL: the images are not downloaded.  Otherwise as in sfmb200_decode_jpeg_batch_scaled.
 * n == 0 does nothing.  sfmb200_orb_last_timings and sfmb200_jpeg_last_stats describe this call; stats [6] counts only the bytes that
 * were downloaded (the error words and statistics, plus the images if asked for).  sfmb200_orb_download_level inspects its last group.
 */
int sfmb200_decode_jpeg_extract_orb(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, int nfeatures,
                                    int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints,
                                    uint8_t* const* out_bgr /* NULL: images not downloaded */, const size_t* out_stride);

/* ---- f-3: PNG and JPEG files, decoded (and downscaled, and ORB-extracted) in one call ----------------------------- */
/*
 * setImagesDirectory collects .jpg and .png files (SfM.cpp:110) and imread reads both.  These calls take any mix of the two formats.
 * PNG output is byte-identical to cv::imread(file, IMREAD_COLOR) with OpenCV 4.13 and libpng 1.6: B,G,R; grey at 1/2/4/8/16 bits,
 * RGB, palette, grey+alpha and RGBA at every legal depth; sub-byte grey scaled to 8 bits (a 1-bit 1 gives 255); 16-bit samples keep
 * their high byte (0x12ff -> 0x12); alpha dropped without compositing; tRNS, gAMA, sRGB, iCCP, sBIT, cHRM ignored; a palette index
 * past the end of PLTE gives (0,0,0); Adam7 interlacing; the EXIF orientation of an eXIf chunk (before or after IDAT) applied --
 * orientations 5-8 swap width and height.  A CRC error in an ancillary chunk drops that chunk (a bad eXIf does not rotate).
 * SFMB200_ERR_INVALID: a CRC error in a critical chunk, no IEND, a truncated file, an invalid zlib header or deflate stream (BTYPE 3,
 * a stored LEN / NLEN mismatch, an over-subscribed or wrongly incomplete code, a bad code-length repeat, a distance before the start),
 * too little image data, a filter type above 4, an Adler-32 mismatch, or any other file cv::imread refuses.  Extra compressed data
 * after the image, or bytes after the zlib stream, still decode.  SFMB200_ERR_UNSUPPORTED: an animated PNG (acTL chunk), more than
 * 65535 files, more than 512 MB of IDAT data in one call, an image with more than 2^31 - 1 bytes of filtered data.  Unlike libpng,
 * nothing is padded or repaired; sfmb200_last_error names the image by its index in the caller's list.
 *
 * The deflate streams decode on the device.  Every bit offset is tested for the start of a dynamic-Huffman block whose header zlib
 * would accept, and every such candidate is decoded to its end-of-block in parallel.  One thread per image then walks the true block
 * sequence from the first block, taking a probed candidate wherever one starts at its position and decoding stored, fixed-Huffman
 * and unprobed blocks itself (a Z_FIXED stream therefore decodes serially: correct, but slower than cv::imread).  Every block is then
 * decoded again in parallel into one word per output byte, and back-references across blocks are resolved by pointer jumping.
 * Unfiltering, Adam7, palette and colour conversion, orientation and the downscale follow on the device.  PNG images run in
 * consecutive groups whose transient device memory (IDAT data, candidates, 5 bytes per filtered byte, block records) stays within
 * SFMB200_PNG_GROUP_BYTES (an image larger than that runs alone); each group makes one upload, one download and one host
 * synchronisation.
 *
 * sfmb200_image_info: host only (no context, no GPU): *format = SFMB200_FORMAT_JPEG or _PNG by signature, the output size after
 * orientation, or the status a decode would return (SFMB200_ERR_INVALID for a file that is neither JPEG nor PNG).
 * sfmb200_decode_images: as sfmb200_decode_jpeg_batch_scaled for any mix of JPEG and PNG files (scale == 1: no downscale).  Every file
 * of both formats is parsed and checked before anything launches.  An all-JPEG list gives exactly the JPEG calls' bytes and
 * statistics.  A mixed list runs one JPEG decode (sfmb200_jpeg_last_stats describes it) and one PNG decode.
 * sfmb200_decode_images_extract_orb: sfmb200_decode_jpeg_extract_orb for any mix of JPEG and PNG files: one ORB pass over all images,
 * in the caller's order, with the same output contract.
 * sfmb200_png_last_stats: the PNG part of the last call, SFMB200_PNG_STATS entries: [0] deflate blocks, [1] blocks the chain took
 * from a probed candidate, [2] blocks the chain decoded itself, [3] candidates probed, [4] resolution rounds run until one changed
 * nothing, summed over groups, [5] bytes uploaded, [6] bytes downloaded, [7] groups, [8] stored blocks, [9] fixed-Huffman blocks.
 */
#define SFMB200_FORMAT_JPEG 1
#define SFMB200_FORMAT_PNG 2
#define SFMB200_PNG_STATS 10
#define SFMB200_PNG_GROUP_BYTES (1ull << 30)
int sfmb200_image_info(const uint8_t* data, size_t size, int* format, int* width, int* height);
int sfmb200_decode_images(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, uint8_t* const* out_bgr,
                          const size_t* out_stride);
int sfmb200_decode_images_extract_orb(sfmb200_ctx* ctx, const uint8_t* const* data, const size_t* size, int n, double scale, int nfeatures,
                                      int max_keypoints, sfmb200_keypoint* keypoints, uint8_t* descriptors, int32_t* n_keypoints,
                                      uint8_t* const* out_bgr /* NULL: images not downloaded */, const size_t* out_stride);
int sfmb200_png_last_stats(const sfmb200_ctx* ctx, int64_t* stats /* [SFMB200_PNG_STATS] */);

/* ---- f-1 on the device: find2D3DMatches and mergeNewPointCloud ------------------------------------------------- */
/*
 * The host code between the stages of SfM::addMoreViewsToReconstruction (SfM.cpp:366-469): find2D3DMatches (:471-528) once per added
 * view and mergeNewPointCloud (:530-600) once per good view, with the results of host/sfm_glue.cpp (which are the reference's).
 *
 * The match matrix lives on the device as a match index.  sfmb200_match_index_create takes the image-pair batch layout without pts
 * (img_off / pairs / match_q / match_t / match_off, the checks of "image-pair batches" above) plus match_d [M], the float distances.
 * The matrix is upper-triangular: every pair must have left < right and appear at most once (SFMB200_ERR_INVALID otherwise); a pair
 * absent from the batch has an empty list, and so has the diagonal: a lookup of a view against itself finds nothing.  At most 1024
 * images, at most INT32_MAX / 4 matches per call.  sfmb200_match_index_set_pair replaces the list of one pair (left < right), as the
 * driver does at SfM.cpp:288 and :431; every later result is that of an index created from the updated matrix.  Destroy an index
 * before its context.  Errors of the three calls below are read with sfmb200_last_error(index's context).
 *
 * A cloud is given as a view list per point: view_off [n + 1] (from 0, monotone), then view_img / view_feat [view_off[n]], the
 * (view, feature) pairs of originatingViews in ascending view order.  A view outside [0, n_img), views not strictly ascending, or a
 * feature outside its view's key points (img_off of the index) is SFMB200_ERR_INVALID with a message; the context stays usable.
 *
 * sfmb200_find_2d3d_matches: for every view v with done[v] == 0, in ascending order, the cloud points that hit v: a point hits at its
 * first originating view (ascending) whose lookup succeeds; for an originating view left of v the first match in list order with
 * queryIdx == its feature, for one right of v the first with trainIdx == its feature, and the hit's feature in v is that match's
 * other index.  out_point / out_feat: cloud index and feature index of every hit, view by view and in cloud order inside a view;
 * view v owns [out_off[v], out_off[v + 1]) (empty for a done view).  The output never exceeds (not-done views) x n_points entries;
 * if out_cap is below out_off[n_img], the call returns SFMB200_ERR_INVALID with out_off filled and nothing else written.
 *
 * sfmb200_merge_point_cloud: mergeNewPointCloud(new points, existing cloud).  Coordinates X [n * 3] float.  Outputs:
 *   outcome [n_new]  SFMB200_MERGE_APPENDED, _MERGED or _DROPPED per new point (in order);
 *   target [n_new]   appended: its index in the merged cloud (n_exist + its rank among the appended points); merged: the cloud index
 *                    of the point the loop broke at (an existing point or an appended one); dropped: -1;
 *   log_* [log_cap]  every `existingPoint.originatingViews[newKv.first] = newKv.second` of the loop, in the order it runs:
 *                    log_target (cloud index), log_view / log_feat (the key and value written; an overwrite of an existing key and a
 *                    key inserted while the same map is iterated are both logged), log_other (the existing key the match confirmed),
 *                    log_pos (its position in the list of pair (min(view, other), max(view, other)): the debug mergeMatchMatrix entry of
 *                    :571).  log_other / log_pos may be NULL.
 *   counts [3]       appended, merged, log entries.
 * The merged cloud is the existing one, then the appended points in order; applying the log in order to it gives the final maps.
 * The log never has more than n_img x new_off[n_new] entries (each view of a new point against at most n_img keys of one map); if
 * log_cap is below counts[2], the call returns SFMB200_ERR_INVALID with counts filled and nothing else written.
 * Each of the three calls makes one host synchronisation (create and set_pair one more when the index grows); same inputs give
 * bitwise-identical outputs.
 */
typedef struct sfmb200_match_index sfmb200_match_index;
enum { SFMB200_MERGE_DROPPED = 0, SFMB200_MERGE_APPENDED = 1, SFMB200_MERGE_MERGED = 2 };
int sfmb200_match_index_create(sfmb200_ctx* ctx, const int32_t* img_off, int n_img, const int32_t* pairs, int n_pairs, const int32_t* match_q,
                               const int32_t* match_t, const float* match_d, const int64_t* match_off, sfmb200_match_index** index);
int sfmb200_match_index_set_pair(sfmb200_match_index* index, int left, int right, const int32_t* match_q, const int32_t* match_t,
                                 const float* match_d, int64_t m);
void sfmb200_match_index_destroy(sfmb200_match_index* index);
int sfmb200_find_2d3d_matches(sfmb200_match_index* index, const uint8_t* done /* [n_img] */, int n_points, const int32_t* view_off,
                              const int32_t* view_img, const int32_t* view_feat, int64_t out_cap, int32_t* out_point, int32_t* out_feat,
                              int64_t* out_off /* [n_img + 1] */);
int sfmb200_merge_point_cloud(sfmb200_match_index* index, int n_exist, const float* X_exist, const int32_t* exist_off, const int32_t* exist_img,
                              const int32_t* exist_feat, int n_new, const float* X_new, const int32_t* new_off, const int32_t* new_img,
                              const int32_t* new_feat, int64_t log_cap, int8_t* outcome, int32_t* target, int32_t* log_target,
                              int32_t* log_view, int32_t* log_feat, int32_t* log_other, int32_t* log_pos, int64_t* counts /* [3] */);

/* ---- multi-GPU plumbing (NCCL, one process per GPU) ------------------------------------------------------ */
#define SFMB200_UNIQUE_ID_BYTES 128
int sfmb200_comm_unique_id(uint8_t* id /* [SFMB200_UNIQUE_ID_BYTES] */);       /* rank 0, then broadcast by the host */
int sfmb200_comm_init(sfmb200_ctx* ctx, const uint8_t* id, int rank, int nranks);
int sfmb200_comm_rank(const sfmb200_ctx* ctx);
int sfmb200_comm_size(const sfmb200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* SFMB200_H */
