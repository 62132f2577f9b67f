"""The device's DLT null vector (csrc/dlt_math.cuh) on both of its paths, through sfmb200_triangulate, sfmb200_triangulate_pairs and
the cheirality test of sfmb200_find_camera_matrices: scenes whose world unit, offset or baseline sends points to the Jacobi
fallback, degenerate two-view geometry, and matches near the epipole.  X is checked against a 40-digit reference on a
sub-sample and against the C oracle and cv2 on every point, under the per-point tolerance of tests/dlt_util.py."""
import numpy as np
import pytest

import dlt_util as du
from essential_util import CX, CY, F, rot
from oracle import cv2_reference
from sfm_toy_library_b200 import capi
from test_gpu_triangulate_pairs import _assert_equal_to_single_calls

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
SWEEP = du.sweep()
BAND = 1e-3           # px: keep may differ from the reprojection test only this close to the 10 px threshold
WORST = {}            # scene -> worst error / tolerance seen on the device (printed with -s)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()
    for k, v in WORST.items():
        print(f"{k}: worst error / tolerance {v:.3f}")


def _matrices(sc):
    return du.triangulation_matrices(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])


def _against(X, A, Xref):
    """error / tolerance of X against another result Xref, with double singular values"""
    return du.error_ratio(X, A, dict(sigma=np.linalg.svd(A, compute_uv=False), X=np.asarray(Xref, np.float64)))


def _reprojection_keep(sc, X):
    """keep as the reprojection of X through cv2's float-rvec round trip decides it, and the points within BAND of 10 px"""
    _, _, err = cv2_reference.triangulate_views(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])   # for its shapes only
    for v, (P, pts) in enumerate(((sc["Pl"], sc["ptsL"]), (sc["Pr"], sc["ptsR"]))):
        rvec, _ = cv2.Rodrigues(np.asarray(P, np.float32)[:, :3].copy())
        with np.errstate(invalid="ignore", over="ignore"):
            proj, _ = cv2.projectPoints(np.asarray(X, np.float32), rvec, np.asarray(P, np.float32)[:, 3].copy(), np.asarray(sc["K"], np.float32), None)
            d = proj.reshape(-1, 2).astype(np.float32) - pts
            err[:, v] = np.sqrt(d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2)
    keep = ~((err[:, 0] > 10.0) | (err[:, 1] > 10.0))
    return keep, err, np.abs(np.max(err, axis=1) - 10.0) < BAND


@pytest.mark.parametrize("name", [n for n, _ in SWEEP])
def test_sweep_against_exact_oracle_and_cv2(ctx, oracle, name):
    sc = dict(SWEEP)[name]
    A = _matrices(sc)
    X, keep, nk = ctx.triangulate(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    assert nk == int(keep.sum())
    idx = du.subsample(len(A), 60)
    r = du.error_ratio(X[idx], A[idx], du.exact(A[idx]))
    Xo, ko, eo = oracle.triangulate(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    Xc, _, _ = cv2_reference.triangulate_views(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    ro, rc = _against(X, A, Xo), _against(X, A, Xc)
    WORST[name] = max(r.max(), ro.max(), rc.max())
    assert r.max() <= 1.0 and ro.max() <= 1.0 and rc.max() <= 1.0, (r.max(), ro.max(), rc.max())
    # keep is what the device's own X reprojects to, and the oracle's keep wherever the two X agree
    kr, _, band = _reprojection_keep(sc, X)
    assert not np.any((keep.astype(bool) != kr) & ~band), np.flatnonzero((keep.astype(bool) != kr) & ~band)[:10]
    same = np.all(X == Xo, axis=1) & ~band & ~(np.abs(np.max(eo, axis=1) - 10.0) < BAND)
    np.testing.assert_array_equal(keep[same], ko[same])


def test_config5_size_all_on_the_fallback(ctx, oracle):
    sc = du.fixture_scaled(100, 1_000_000, seed=5)
    A = _matrices(sc)
    _, ok, _ = du.host_null_vectors(A)
    assert (du.path(du.gate_margin(A), ok) == "fallback").all()
    X, keep, nk = ctx.triangulate(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    assert nk == int(keep.sum()) > 0.9e6
    Xo, ko, eo = oracle.triangulate(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    r = _against(X, A, Xo)
    WORST["fixture x100, 1 M points"] = r.max()
    assert r.max() <= 1.0, r.max()
    same = np.all(X == Xo, axis=1) & ~(np.abs(np.max(eo, axis=1) - 10.0) < BAND)
    np.testing.assert_array_equal(keep[same], ko[same])
    X2, keep2, nk2 = ctx.triangulate(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    np.testing.assert_array_equal(X2, X); np.testing.assert_array_equal(keep2, keep); assert nk2 == nk


@pytest.mark.parametrize("scene", ["fixture x10", "baseline 0.0001 depth 3 forward"])
def test_mixed_warps_give_the_same_bits_in_any_company(ctx, scene):
    sc = dict(SWEEP)[scene]
    _, ok, _ = du.host_null_vectors(_matrices(sc))
    w = ok[: len(ok) // 32 * 32].reshape(-1, 32)
    assert (w.any(1) & ~w.all(1)).sum() >= 5                  # warps whose lanes take different paths
    args = (sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])
    X, keep, _ = ctx.triangulate(*args)
    for sel in (np.flatnonzero(ok), np.flatnonzero(~ok)):
        Xs, ks, _ = ctx.triangulate(*args, sel.astype(np.int32), sel.astype(np.int32))
        np.testing.assert_array_equal(Xs, X[sel]); np.testing.assert_array_equal(ks, keep[sel])
    for i in range(len(ok)):
        Xi, ki, _ = ctx.triangulate(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"][i:i + 1], sc["ptsR"][i:i + 1])
        assert np.array_equal(Xi[0], X[i]) and ki[0] == keep[i], i


def test_pairs_mixing_both_paths_equal_their_single_calls(ctx):
    scenes = [du.fixture_scaled(1, 3000, seed=1), du.fixture_scaled(100, 3000, seed=2), dict(SWEEP)["identical"],
              du.fixture_scaled(1, 10, seed=3), dict(SWEEP)["fixture x10"], dict(SWEEP)["epipole 0.01 px"]]
    sizes = [3000, 3000, 1000, 0, 2000, 500]
    pts, pairs, poses, mq, mt = [], [], [], [], []
    for sc, m in zip(scenes, sizes):
        pairs.append((len(pts), len(pts) + 1)); pts += [sc["ptsL"], sc["ptsR"]]; poses.append((sc["Pl"], sc["Pr"]))
        mq.append(np.arange(m)); mt.append(np.arange(m))
    q, t, off = capi.flatten_matches(mq, mt)
    args = (du.K, np.array(poses), pts, np.array(pairs), q, t, off)
    out = ctx.triangulate_pairs(*args)
    assert out[2][3] == 0
    _assert_equal_to_single_calls(ctx, *args, out)
    args = (du.K, np.array(poses[::-1]), pts, np.array(pairs[::-1]), *capi.flatten_matches(mq[::-1], mt[::-1]))
    _assert_equal_to_single_calls(ctx, *args, ctx.triangulate_pairs(*args))


# ---------------------------------------------------------------- recoverPose's cheirality test near the epipole
KE = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1]], np.float32)


def _pose_scene(kind, seed):
    """noise-free matches (float32 pixels), so that the estimated epipole is the principal point to far below 0.01 px: forward
    motion with 150 matches 0.01-0.5 px from the epipole and 4 exactly at it among 600 ordinary points, or a near-pure rotation
    (|t| = 0.1 at depths 3..10: in recoverPose's unit |t| = 1 the depths straddle its distance threshold of 50)"""
    rs = np.random.RandomState(seed)
    n = 600
    X = np.c_[rs.uniform(-10, 10, n), rs.uniform(-7.5, 7.5, n), rs.uniform(3, 10, n)]
    if kind == "forward":
        R, t = rot([0, 0, 0]), np.array([0.0, 0.0, -1.0])
        d = rs.uniform(3, 10, 150); r = np.exp(rs.uniform(np.log(0.01), np.log(0.5), 150)) / F * d; ang = rs.uniform(0, 2 * np.pi, 150)
        Xe = np.c_[r * np.cos(ang), r * np.sin(ang), d]
    else:
        R, t = rot([0.02, 0.1, 0.0]), 0.1 * np.array([0.6, 0.0, 0.8])
        Xe = np.zeros((0, 3))

    def px(P, Y):
        Yc = Y @ P[:, :3].T + P[:, 3]
        return np.c_[F * Yc[:, 0] / Yc[:, 2] + CX, F * Yc[:, 1] / Yc[:, 2] + CY]
    P0, P1 = np.c_[np.eye(3), np.zeros(3)], np.c_[R, t]
    a = px(P0, X); b = px(P1, X)
    a = np.r_[a, px(P0, Xe)]; b = np.r_[b, px(P1, Xe)]
    if kind == "forward":
        at = np.tile([CX, CY], (4, 1))
        a = np.r_[a, at]; b = np.r_[b, at]
    return a.astype(np.float32), b.astype(np.float32)


def _depth_tests_near_threshold(E, R, t, a, b, dist=50.0):
    """per match: does one of recoverPose's depth tests (Q2 Q3 > 0, z < dist, 0 < z2 < dist) lie within the conditioning bound
    of its threshold?  The bound is that of tests/dlt_util.py: delta n (1 + |X|) on the dehomogenised point"""
    Pc = np.c_[R, t]
    A = du.cheirality_matrices(a, b, F, CX, CY, Pc)
    _, s, Vt = np.linalg.svd(A)
    Q = Vt[:, 3, :]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        delta = 16 * du.U53 * s[:, 0] / (s[:, 2] - s[:, 3]) + 1e-12
        X = Q[:, :3] / Q[:, 3:4]
        nx = np.linalg.norm(X, axis=1)
        tol = delta * np.sqrt(1 + nx ** 2) * (1 + nx) * 4
        z = X[:, 2]; z2 = X @ R[2] + t[2]
        near = (np.abs(Q[:, 2]) <= 4 * delta) | (np.abs(Q[:, 3]) <= 4 * delta)
        near |= (np.abs(z - dist) <= tol) | (np.abs(z2) <= tol) | (np.abs(z2 - dist) <= tol)
    return near | ~np.isfinite(tol) | (s[:, 2] - s[:, 3] <= du.RANK_DEFICIENT * s[:, 0])


@pytest.mark.parametrize("kind,seed", [("forward", 0), ("forward", 1), ("rotation", 2)])
def test_recover_pose_near_the_epipole(ctx, kind, seed):
    a, b = _pose_scene(kind, seed)
    E, R, t, inl, pm, s = ctx.find_camera_matrices(KE, a, b, seed=seed)
    assert s["found"]
    n, Rc, tc, mc = cv2.recoverPose(E, a.astype(np.float64), b.astype(np.float64), focal=F, pp=(CX, CY), mask=inl.reshape(-1, 1).copy())
    np.testing.assert_allclose(R, Rc, rtol=0, atol=1e-9); np.testing.assert_allclose(t, tc.ravel(), rtol=0, atol=1e-9)
    diff = (pm != 0) != (mc.ravel() != 0)
    near = _depth_tests_near_threshold(E, R, t, a, b)
    assert not np.any(diff & ~near), np.flatnonzero(diff & ~near)
    assert s["n_good"] == int(pm.sum())
    # the fallback really ran: at least 50 inlier cheirality solves lie 100x below the closed form's gate
    sel = inl.astype(bool)
    R1, R2, tt = cv2.decomposeEssentialMat(E)
    n_fallback = 0
    for Rk, tk in ((R1, tt), (R2, tt), (R1, -tt), (R2, -tt)):
        A = du.cheirality_matrices(a[sel], b[sel], F, CX, CY, np.c_[Rk, tk.ravel()])
        _, ok, _ = du.host_null_vectors(A)
        n_fallback += int((du.path(du.gate_margin(A), ok) == "fallback").sum())
    if kind == "forward":
        assert n_fallback >= 50, n_fallback
        # matches exactly at the principal point, x1 = x2 = 0: the Sampson error is E22^2 / (E02^2 + E12^2 + E20^2 + E21^2), a ratio
        # of E's rounding errors for forward motion (0/0 when they vanish, and NaN is no inlier).  The device decides it exactly as
        # this double evaluation does.
        e = E.reshape(-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            samp = np.float32(e[8] * e[8] / (e[2] * e[2] + e[5] * e[5] + e[6] * e[6] + e[7] * e[7]))
        assert (inl[-4:] != 0).tolist() == [bool(samp <= np.float32((1.0 / F) ** 2))] * 4, samp


@pytest.mark.parametrize("kind", ["forward", "rotation"])
def test_pose_pairs_equal_single_calls_near_the_epipole(ctx, kind):
    scenes = [_pose_scene(kind, s) for s in range(3)]
    pts, pairs = [], []
    for a, b in scenes:
        pairs.append((len(pts), len(pts) + 1)); pts += [a, b]
    q, t, off = capi.flatten_matches([np.arange(len(a)) for a, _ in scenes], [np.arange(len(a)) for a, _ in scenes])
    E, R, T, inl, pm, s = ctx.find_camera_matrices_pairs(KE, pts, np.array(pairs), q, t, off, seed=7)
    for p, (a, b) in enumerate(scenes):
        E1, R1, t1, inl1, pm1, s1 = ctx.find_camera_matrices(KE, a, b, seed=7)
        sl = slice(int(off[p]), int(off[p + 1]))
        np.testing.assert_array_equal(E[p], E1); np.testing.assert_array_equal(R[p], R1); np.testing.assert_array_equal(T[p], t1)
        np.testing.assert_array_equal(inl[sl], inl1); np.testing.assert_array_equal(pm[sl], pm1)
        assert s["n_good"][p] == s1["n_good"] and s["n_inliers"][p] == s1["n_inliers"]
