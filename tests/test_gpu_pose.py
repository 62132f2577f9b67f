"""sfmb200_find_camera_pose (csrc/pose.cu): findCameraPoseFrom2D3DMatch's cv::solvePnPRansac on the device.  The RANSAC draws its own
seeded samples, so it is compared with cv2 statistically; what can be exact is checked exactly: the trace replays through
sfmb200_ransac_score and the restatement of OpenCV's selection, and the refit lands on cv2.solvePnP(ITERATIVE)'s least-squares
minimum over the same inliers."""
import ctypes as C

import numpy as np
import pytest

from cfg1_util import Cfg1
import essential_oracle as eo
from sfm_toy_library_b200 import capi, ransac, runsfm, stages, synth

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cfg1():
    return Cfg1()


def pnp_set(cfg, k):
    """PnP call k of the crazyhorse replay: 3D points, 2D points, the intrinsics of that moment (the bundle adjustment before it
    refines the focal length), cv2's accept decision and pose."""
    g = cfg.g
    return (g[f"pnp_{k}_p3"], g[f"pnp_{k}_p2"], np.asarray(g[f"ba_{k}_K_after"], np.float32), bool(g[f"pnp_{k}_ok"]),
            g[f"pnp_{k}_pose"].astype(np.float64))


def synthetic_set(n, outliers, seed, noise=0.5):
    rs = np.random.RandomState(seed)
    K = np.array([[1200, 0, 640], [0, 1150, 360], [0, 0, 1]], np.float32)
    R = synth.angle_axis_to_rotmat(rs.normal(0, 0.3, 3)); t = np.array([0.3, -0.2, 6.0]) + rs.normal(0, 0.2, 3)
    Xc = np.c_[rs.uniform(-3, 3, (n, 2)), rs.uniform(4, 12, n)]
    X = (Xc - t) @ R
    uv = Xc[:, :2] / Xc[:, 2:] * [K[0, 0], K[1, 1]] + K[:2, 2] + rs.normal(0, noise, (n, 2))
    bad = rs.uniform(size=n) < outliers
    uv[bad] = rs.uniform([0, 0], [1280, 720], (int(bad.sum()), 2))
    return X.astype(np.float32), uv.astype(np.float32), K, R, t


def test_trace_replays_through_ransac_score_and_sequential_select(ctx, cfg1):
    for k in range(cfg1.n_pnp):
        X, uv, K, _, _ = pnp_set(cfg1, k)
        _, R0, t0, mask0, s0 = ctx.find_camera_pose(K, X, uv, seed=k, refine_iters=0)
        samples, counts = ctx.pose_last_trace()
        assert samples.shape == (100, 5) and s0["n_samples"] == 100
        Rt, ok = ctx.epnp(X[samples].astype(np.float64), uv[samples].astype(np.float64), K.astype(np.float64))
        np.testing.assert_array_equal(ok.astype(bool), counts >= 0)
        assert s0["n_hypotheses"] == int(ok.sum())
        rc, _, _ = ctx.ransac_score(capi.MODEL_POSE, X, uv, Rt[ok == 1].reshape(-1, 12), K.reshape(-1), 10.0, want_mask=False)
        np.testing.assert_array_equal(rc, counts[ok == 1])              # bitwise the device's own scoring
        best, good, it = eo.sequential_select(ok.astype(np.int32), counts[ok == 1], len(X), max_iters=100, confidence=0.99, model_points=5)
        assert best >= 0 and s0["found"] == 1 and good == s0["n_inliers"] and it == s0["iterations"], (k, best, good, it, s0)
        win = np.flatnonzero(ok)[best]
        np.testing.assert_array_equal(R0, Rt[win][:, :3]); np.testing.assert_array_equal(t0, Rt[win][:, 3])
        _, _, m2 = ctx.ransac_score(capi.MODEL_POSE, X, uv, Rt[win].reshape(1, 12), K.reshape(-1), 10.0)
        np.testing.assert_array_equal(mask0, m2)
        assert int(mask0.sum()) == s0["n_inliers"]
        # the refit keeps the RANSAC winner's mask and count
        _, _, _, mask, s = ctx.find_camera_pose(K, X, uv, seed=k)
        np.testing.assert_array_equal(mask, mask0)
        assert s["n_inliers"] == s0["n_inliers"] and s["iterations"] == s0["iterations"]


def _refit_matches_cv2(ctx, K, X, uv, seed):
    rv, R, t, mask, s = ctx.find_camera_pose(K, X, uv, seed=seed)
    _, R0, t0, mask0, _ = ctx.find_camera_pose(K, X, uv, seed=seed, refine_iters=0)
    assert s["found"] and s["refined"] == 1, s
    np.testing.assert_array_equal(mask, mask0)
    sel = mask.astype(bool)
    r0, _ = cv2.Rodrigues(R0)
    ok, rvc, tvc = cv2.solvePnP(X[sel].astype(np.float64), uv[sel].astype(np.float64), K.astype(np.float64), None, r0, t0.reshape(3, 1).copy(),
                                True, cv2.SOLVEPNP_ITERATIVE)
    assert ok
    Rc, _ = cv2.Rodrigues(rvc)
    assert np.abs(R - Rc).max() <= 1e-6, (np.abs(R - Rc).max(), s)
    assert np.abs(t - tvc.ravel()).max() <= 1e-6 * np.linalg.norm(t), (t, tvc.ravel())
    Rr, _ = cv2.Rodrigues(rv)
    assert np.abs(Rr - R).max() < 1e-12                                  # R = Rodrigues(rvec)


def test_refit_is_the_least_squares_minimum_crazyhorse(ctx, cfg1):
    for k in range(cfg1.n_pnp):
        X, uv, K, _, _ = pnp_set(cfg1, k)
        _refit_matches_cv2(ctx, K, X, uv, seed=3)


@pytest.mark.parametrize("n,outliers,seed", [(60, 0.0, 1), (500, 0.3, 2), (5000, 0.5, 3)])
def test_refit_is_the_least_squares_minimum_synthetic(ctx, n, outliers, seed):
    X, uv, K, Rtrue, ttrue = synthetic_set(n, outliers, seed)
    _refit_matches_cv2(ctx, K, X, uv, seed=seed)
    _, R, t, mask, s = ctx.find_camera_pose(K, X, uv, seed=seed)
    assert np.abs(R - Rtrue).max() < 5e-3 and np.abs(t - ttrue).max() < 5e-2, (R, Rtrue, t, ttrue)


def _host_path(K, X, uv, seed):
    """The hypotheses of the existing host path (ransac.findCameraPoseFrom2D3DMatch: cv2 EPnP on seeded samples, GPU scoring, cv2
    refit) for one seed."""
    Kd = K.astype(np.float64)
    hyps = ransac.pose_hypotheses(X, uv, Kd, 100, np.random.RandomState(seed))
    return hyps, Kd


def test_agreement_with_cv2_within_the_host_paths_spread(ctx, cfg1):
    """The yardstick is the existing host path's hypotheses (cv2 EPnP on seeded samples) over seeds 0-31, selected with OpenCV's
    rule and refitted by cv2: the device's typical inlier count and distance to cv2's pose must fall inside that spread."""
    for k in range(cfg1.n_pnp):
        X, uv, K, ok_ref, pose_ref = pnp_set(cfg1, k)
        intr = stages.Intrinsics(K.copy())
        n_h, dR_h, dt_h = [], [], []
        for seed in range(32):
            hyps, Kd = _host_path(K, X, uv, seed)
            counts, _, _ = ctx.ransac_score(capi.MODEL_POSE, X, uv, hyps, Kd.reshape(-1), 10.0, want_mask=False)
            # the host path keeps the best of all its samples; OpenCV's loop (and the device) stop at the adaptive budget, so the
            # host path's samples go through that loop, and cv2 refits the pose it keeps on that pose's inliers
            win, good, _ = eo.sequential_select(np.ones(len(counts), np.int32), counts, len(X), max_iters=100, confidence=0.99, model_points=5)
            _, _, mask = ctx.ransac_score(capi.MODEL_POSE, X, uv, hyps[win:win + 1], Kd.reshape(-1), 10.0)
            P = hyps[win].reshape(3, 4); sel = mask.astype(bool)
            r0, _ = cv2.Rodrigues(P[:, :3].copy())
            _, rv, tv = cv2.solvePnP(X[sel].astype(np.float64), uv[sel].astype(np.float64), Kd, None, r0, P[:, 3].reshape(3, 1).copy(), True,
                                     cv2.SOLVEPNP_ITERATIVE)
            pose = np.c_[cv2.Rodrigues(rv)[0], tv.reshape(3)].astype(np.float32)
            n_h.append(good)
            dR_h.append(np.abs(pose[:, :3] - pose_ref[:, :3]).max()); dt_h.append(np.abs(pose[:, 3] - pose_ref[:, 3]).max())
        # the device over the same 32 seeds: every decision cv2's, and its typical (median) result inside the host path's spread
        n_d, dR_d, dt_d = [], [], []
        for seed in range(32):
            okd, pose = ransac.findCameraPoseFrom2D3DMatch_gpu(intr, uv, X, ctx=ctx, seed=seed)
            assert okd == ok_ref, (k, seed)
            n_d.append(ctx.find_camera_pose(K, X, uv, seed=seed)[4]["n_inliers"])
            dR_d.append(np.abs(pose[:, :3] - pose_ref[:, :3]).max()); dt_d.append(np.abs(pose[:, 3] - pose_ref[:, 3]).max())
        assert min(n_h) <= np.median(n_d) <= len(X), (k, n_d, min(n_h), max(n_h))
        assert np.median(dR_d) <= max(dR_h), (k, np.median(dR_d), max(dR_h))
        assert np.median(dt_d) <= max(dt_h), (k, np.median(dt_d), max(dt_h))


def test_reference_unit_test_scene(ctx):
    # the reference's find_camera_pose_from_2d3d_match (SfMUnitTests.cpp:194-216): 12 exact correspondences, R to 0.01, t to 0.1
    Pl, _ = synth.fixture_poses()
    rvec, _ = cv2.Rodrigues(Pl[:, :3].copy())
    proj, _ = cv2.projectPoints(synth.CANNED_POINTS, rvec, Pl[:, 3].copy(), synth.TEST_K, None)
    ok, pose = ransac.findCameraPoseFrom2D3DMatch_gpu(stages.Intrinsics(synth.TEST_K), proj.reshape(-1, 2).astype(np.float32), synth.CANNED_POINTS,
                                                      ctx=ctx)
    assert ok
    assert np.abs(pose[:, :3] - Pl[:, :3]).max() < 0.01 and np.abs(pose[:, 3] - Pl[:, 3]).max() < 0.1


def test_determinism_and_seeds(ctx):
    X, uv, K, _, _ = synthetic_set(3000, 0.3, 7)
    a = ctx.find_camera_pose(K, X, uv, seed=11); ta = ctx.pose_last_trace()
    b = ctx.find_camera_pose(K, X, uv, seed=11); tb = ctx.pose_last_trace()
    for x, y in zip(a[:4] + ta, b[:4] + tb):
        np.testing.assert_array_equal(x, y)
    assert a[4] == b[4]
    ctx.find_camera_pose(K, X, uv, seed=12); tc = ctx.pose_last_trace()
    assert (tc[0] != ta[0]).any(axis=1).mean() > 0.9


def test_edge_cases(ctx):
    X, uv, K, R, t = synthetic_set(40, 0.0, 8, noise=0.0)
    # m < 5: nothing found, zero outputs, no trace
    for m in (0, 1, 4):
        rv, Rm, tm, mask, s = ctx.find_camera_pose(K, X[:m], uv[:m])
        assert s["found"] == 0 and s["n_samples"] == 0 and not Rm.any() and not tm.any() and not rv.any() and not mask.any()
        assert ctx.pose_last_trace()[0].shape == (0, 5)
    # m == 5: EPnP on the five points, every point an inlier, no refit
    rv, Rm, tm, mask, s = ctx.find_camera_pose(K, X[:5], uv[:5])
    assert s["found"] == 1 and s["n_inliers"] == 5 and s["refined"] == 0 and s["n_samples"] == 1 and mask.all()
    assert np.abs(Rm - R).max() < 1e-4 and np.abs(tm - t).max() < 1e-3
    # all outliers: no pose passes the reference's ratio test
    rs = np.random.RandomState(9)
    Xo = rs.uniform(-5, 5, (300, 3)).astype(np.float32) + [0, 0, 20]; uvo = rs.uniform(0, 1280, (300, 2)).astype(np.float32)
    ok, _ = ransac.findCameraPoseFrom2D3DMatch_gpu(stages.Intrinsics(K), uvo, Xo, ctx=ctx)
    assert not ok
    _, _, _, mask, s = ctx.find_camera_pose(K, Xo, uvo)
    assert int(mask.sum()) == s["n_inliers"] and (s["found"] == 0 or s["n_inliers"] < 150)
    # non-finite correspondences are never inliers and do not disturb the others
    Xn = X.copy(); uvn = uv.copy(); Xn[3, 1] = np.nan; uvn[7, 0] = np.inf
    _, Rn, tn, mask, s = ctx.find_camera_pose(K, Xn, uvn)
    assert s["found"] == 1 and mask[3] == 0 and mask[7] == 0 and s["n_inliers"] == 38
    assert np.all(np.isfinite(Rn)) and np.abs(Rn - R).max() < 1e-5
    # refused arguments: non-finite K, fx or fy <= 0, bad options
    for q, v in ((0, np.nan), (5, np.inf), (0, 0.0), (4, -1150.0)):
        Kb = K.copy().reshape(9); Kb[q] = v
        with pytest.raises(capi.SfmB200Error):
            ctx.find_camera_pose(Kb, X, uv)
    for kw in ({"max_iters": 0}, {"confidence": 1.0}, {"confidence": 0.0}, {"threshold_px": 0.0}, {"threshold_px": float("inf")},
               {"refine_iters": -1}):
        with pytest.raises(capi.SfmB200Error):
            ctx.find_camera_pose(K, X, uv, **kw)
    # the context stays usable, and every output may be NULL
    full = ctx.find_camera_pose(K, X, uv, seed=5)
    L = capi.lib()
    Kc = np.ascontiguousarray(K.reshape(9)); Xc = np.ascontiguousarray(X); uc = np.ascontiguousarray(uv)
    f = C.POINTER(C.c_float)
    assert L.sfmb200_find_camera_pose(ctx._h, Kc.ctypes.data_as(f), Xc.ctypes.data_as(f), uc.ctypes.data_as(f), len(X), None, None, None, None, None,
                                      None) == 0
    s = capi.PoseSummary(); t3 = np.zeros(3)
    o = capi.pose_default_options(seed=5)
    assert L.sfmb200_find_camera_pose(ctx._h, Kc.ctypes.data_as(f), Xc.ctypes.data_as(f), uc.ctypes.data_as(f), len(X), C.byref(o), None, None,
                                      t3.ctypes.data_as(C.POINTER(C.c_double)), None, C.byref(s)) == 0
    np.testing.assert_array_equal(t3, full[2]); assert s.as_dict() == full[4]
    assert L.sfmb200_find_camera_pose(ctx._h, None, Xc.ctypes.data_as(f), uc.ctypes.data_as(f), len(X), None, None, None, None, None, None) != 0
    assert L.sfmb200_find_camera_pose(ctx._h, Kc.ctypes.data_as(f), None, uc.ctypes.data_as(f), len(X), None, None, None, None, None, None) != 0


def test_whole_crazyhorse_replay(ctx, cfg1):
    sfm = runsfm.SfM(cfg1.features, cfg1.size,
                     matchAllPairs=lambda f, pr: stages.matchAllPairs(f, pr, ctx=ctx), matchFeatures=lambda a, b: stages.matchFeatures(a, b, ctx=ctx),
                     triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx), adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx),
                     findHomographyInliers=lambda *a: ransac.findHomographyInliers_gpu(*a, ctx=ctx),
                     findCameraMatricesFromMatch=lambda *a: ransac.findCameraMatricesFromMatch_gpu(*a, ctx=ctx),
                     findCameraPoseFrom2D3DMatch=lambda *a: ransac.findCameraPoseFrom2D3DMatch_gpu(*a, ctx=ctx))
    sfm.runSfM()
    assert len(sfm.mDoneViews) == 7
    assert 0.5 * len(cfg1.g["final_cloud"]) < len(sfm.mReconstructionCloud) < 2.0 * len(cfg1.g["final_cloud"])
    assert abs(float(sfm.mIntrinsics.K[0, 0]) - float(cfg1.g["final_K"][0, 0])) < 0.15 * float(cfg1.g["final_K"][0, 0])
