"""Host side of SURVEY.md 8 row f-2: the reference's three RANSAC stages (SfMStereoUtilities.cpp:51-72, :74-118, :208-243) with
the hypothesis SCORING on the GPU (sfmb200_ransac_score: every hypothesis of a run against every correspondence in one launch
sequence) and the hypothesis GENERATION on the host through OpenCV's own minimal solvers (cv2.getPerspectiveTransform: 4 points;
cv2.findEssentialMat on exactly 5 points = the five-point solver, all its solutions; cv2.solvePnP(EPNP) on 5 points, what
cv::solvePnPRansac uses for its minimal sets).  Same names / argument meaning as the reference functions, so they plug into the
driver mirror (runsfm.SfM(findHomographyInliers=..., ...)).

Parity: per hypothesis the inlier set is OpenCV's (same error formula, same arithmetic type, same threshold rule; tests/
test_gpu_ransac.py checks it against the restatement pinned to cv2).  The RANSAC outcome as a whole is only statistically
comparable -- cv:: draws its samples from its own RNG and stops adaptively; here a fixed number of seeded samples is scored.
"""
import numpy as np

from . import capi
from .stages import Features, Intrinsics, default_context

RANSAC_THRESHOLD = 10.0                # SfMStereoUtilities.cpp:41
POSE_INLIERS_MINIMAL_RATIO = 0.5       # SfMCommon.h:53


def _samples(rng, n, k, count):
    """`count` index sets of k distinct correspondences."""
    out = np.empty((count, k), np.int64)
    for i in range(count):
        out[i] = rng.choice(n, k, replace=False)
    return out


def homography_hypotheses(a, b, count, rng):
    import cv2
    hyps = []
    for idx in _samples(rng, len(a), 4, count):
        H = cv2.getPerspectiveTransform(np.ascontiguousarray(a[idx]), np.ascontiguousarray(b[idx]))
        if np.all(np.isfinite(H)) and abs(H[2, 2]) > 1e-12:
            hyps.append(H / H[2, 2])
    return np.array(hyps).reshape(-1, 9)


def essential_hypotheses(a, b, focal, pp, count, rng):
    import cv2
    hyps = []
    for idx in _samples(rng, len(a), 5, count):
        E, _ = cv2.findEssentialMat(np.ascontiguousarray(a[idx]), np.ascontiguousarray(b[idx]), focal, pp, cv2.RANSAC, 0.999, 1.0)
        if E is None:
            continue
        for k in range(E.shape[0] // 3):                   # the five-point solver returns up to 10 solutions, stacked
            hyps.append(E[3 * k:3 * k + 3].reshape(-1))
    return np.array(hyps).reshape(-1, 9)


def pose_hypotheses(X, uv, K, count, rng):
    import cv2
    hyps = []
    for idx in _samples(rng, len(X), 5, count):
        ok, rvec, tvec = cv2.solvePnP(np.ascontiguousarray(X[idx], np.float64), np.ascontiguousarray(uv[idx], np.float64), K.astype(np.float64), None, flags=cv2.SOLVEPNP_EPNP)
        if ok and np.all(np.isfinite(rvec)) and np.all(np.isfinite(tvec)):
            R, _ = cv2.Rodrigues(rvec)
            hyps.append(np.concatenate([R, tvec.reshape(3, 1)], 1).reshape(-1))
    return np.array(hyps).reshape(-1, 12)


def findHomographyInliers(left: Features, right: Features, matches, ctx=None, iterations=256, seed=0):
    """SfMStereoUtilities::findHomographyInliers (SfMStereoUtilities.cpp:51-72): number of inliers of the best homography."""
    if len(matches) < 4:
        return 0
    ctx = ctx or default_context()
    a = left.points[matches["queryIdx"]]; b = right.points[matches["trainIdx"]]
    hyps = homography_hypotheses(a, b, iterations, np.random.RandomState(seed))
    if len(hyps) == 0:
        return 0
    counts, best, _ = ctx.ransac_score(capi.MODEL_HOMOGRAPHY, a, b, hyps, None, RANSAC_THRESHOLD, want_mask=False)
    return int(counts[best])


def homographyInliersAllPairs(features, pairs, matches, ctx=None):
    """findHomographyInliers (SfMStereoUtilities.cpp:51-72) for every pair in one device call (sfmb200_find_homography_pairs):
    cv::findHomography(RANSAC, RANSAC_THRESHOLD)'s own sample sequence, selection and refinement, so the counts are the
    reference's.  features: per image Features; pairs [(i, j), ...]; matches: per pair a structured array with queryIdx / trainIdx.
    Returns the inlier counts [len(pairs)] (0 for fewer than 4 matches or no model)."""
    ctx = ctx or default_context()
    if len(pairs) == 0:
        return np.zeros(0, np.int64)
    off = np.zeros(len(pairs) + 1, np.int64); off[1:] = np.cumsum([len(m) for m in matches])
    mq = np.concatenate([np.asarray(m["queryIdx"], np.int32) for m in matches]); mt = np.concatenate([np.asarray(m["trainIdx"], np.int32) for m in matches])
    _, _, s = ctx.find_homography_pairs([f.points for f in features], pairs, mq, mt, off, threshold_px=RANSAC_THRESHOLD)
    return np.where(s["found"] != 0, s["n_inliers"], 0).astype(np.int64)


def findHomographyInliers_gpu(left: Features, right: Features, matches, ctx=None):
    """SfMStereoUtilities::findHomographyInliers (SfMStereoUtilities.cpp:51-72) on the device: countNonZero of the mask
    cv::findHomography(RANSAC, RANSAC_THRESHOLD) returns, 0 for fewer than 4 matches or no model."""
    return int(homographyInliersAllPairs([left, right], [(0, 1)], [matches], ctx)[0])


def findCameraMatricesFromMatch(intrinsics: Intrinsics, matches, left: Features, right: Features, ctx=None, iterations=200, seed=0):
    """SfMStereoUtilities::findCameraMatricesFromMatch (SfMStereoUtilities.cpp:74-118).  Returns (success, prunedMatches, Pleft, Pright)."""
    import cv2
    ctx = ctx or default_context()
    K = intrinsics.K
    focal = float(K[0, 0]); pp = (float(K[0, 2]), float(K[1, 2]))
    a = left.points[matches["queryIdx"]]; b = right.points[matches["trainIdx"]]
    Pleft = np.eye(3, 4, dtype=np.float32)
    if len(a) < 5:
        return False, matches[:0].copy(), Pleft, Pleft.copy()
    hyps = essential_hypotheses(a, b, focal, pp, iterations, np.random.RandomState(seed))
    if len(hyps) == 0:
        return False, matches[:0].copy(), Pleft, Pleft.copy()
    counts, best, mask = ctx.ransac_score(capi.MODEL_ESSENTIAL, a, b, hyps, (focal, pp[0], pp[1]), 1.0 / focal)
    E = hyps[best].reshape(3, 3)
    m = mask.reshape(-1, 1).copy()
    _, R, t, m = cv2.recoverPose(E, a, b, focal=focal, pp=pp, mask=m)                     # cheirality, like the reference (:92)
    Pright = np.concatenate([R, t.reshape(3, 1)], 1).astype(np.float32)
    return True, matches[m.reshape(-1) != 0].copy(), Pleft, Pright


def findCameraMatricesFromMatch_gpu(intrinsics: Intrinsics, matches, left: Features, right: Features, ctx=None, seed=0):
    """SfMStereoUtilities::findCameraMatricesFromMatch (SfMStereoUtilities.cpp:74-118) entirely on the device
    (sfmb200_find_camera_matrices: five-point samples, scoring, OpenCV's sequential selection, recoverPose).
    Returns (success, prunedMatches, Pleft, Pright) like the reference."""
    ctx = ctx or default_context()
    Pleft = np.eye(3, 4, dtype=np.float32)
    E, R, t, _, pose_mask, s = ctx.find_camera_matrices(intrinsics.K, left.points, right.points, matches["queryIdx"], matches["trainIdx"], seed=seed)
    if not s["found"]:
        return False, matches[:0].copy(), Pleft, Pleft.copy()
    Pright = np.concatenate([R, t.reshape(3, 1)], 1).astype(np.float32)           # :105-107
    return True, matches[pose_mask != 0].copy(), Pleft, Pright


def findCameraPoseFrom2D3DMatch(intrinsics: Intrinsics, points2D, points3D, ctx=None, iterations=100, seed=0):
    """SfMStereoUtilities::findCameraPoseFrom2D3DMatch (SfMStereoUtilities.cpp:208-243).  Returns (success, pose 3x4 float32)."""
    import cv2
    ctx = ctx or default_context()
    K = np.asarray(intrinsics.K, np.float64)
    n = len(points2D)
    if n < 5:
        return False, None
    hyps = pose_hypotheses(points3D, points2D, K, iterations, np.random.RandomState(seed))
    if len(hyps) == 0:
        return False, None
    counts, best, mask = ctx.ransac_score(capi.MODEL_POSE, points3D, points2D, hyps, K.reshape(-1), RANSAC_THRESHOLD)
    if np.float32(counts[best]) / np.float32(n) < POSE_INLIERS_MINIMAL_RATIO:            # :231-234
        return False, None
    P = hyps[best].reshape(3, 4)
    sel = mask.astype(bool)
    if sel.sum() >= 6:                                      # cv::solvePnPRansac refits on the inliers of the best model
        rvec, _ = cv2.Rodrigues(P[:, :3]); tvec = P[:, 3].reshape(3, 1).copy()
        ok, rvec, tvec = cv2.solvePnP(points3D[sel].astype(np.float64), points2D[sel].astype(np.float64), K, None, rvec, tvec, True, cv2.SOLVEPNP_ITERATIVE)
        if ok:
            R, _ = cv2.Rodrigues(rvec); P = np.concatenate([R, tvec.reshape(3, 1)], 1)
    return True, P.astype(np.float32)
