"""Essential-matrix RANSAC and pose recovery on the device (sfmb200_find_camera_matrices, SfMStereoUtilities.cpp:74-118).
The five-point solver against cv2 on the same samples; every per-solution count against the scoring restatement; the selection
against the oracle's replay of OpenCV's sequential loop; the pose against cv2.recoverPose on the returned E and mask; the whole
RANSAC against cv2 statistically; the runSfM replay with the device stage."""
import numpy as np
import pytest

from cfg1_util import Cfg1
import essential_oracle as eo
from essential_util import CX, CY, F, compare_with_cv2, five_point_samples, synthetic_scene
from oracle import ransac_oracle as ro
from sfm_toy_library_b200 import capi, ransac, runsfm, stages

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
K = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1]], np.float32)
AUX = (F, CX, CY)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cfg1():
    return Cfg1()


def _pair(cfg1, p):
    i, j = cfg1.pairs[p]; q, t, _ = cfg1.matches[p]
    return cfg1.features[i].points[q], cfg1.features[j].points[t]


def _angle(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


def test_device_five_point_matches_cv2(ctx, cfg1):
    x1, x2, A, B = five_point_samples(cfg1)
    E, n = ctx.five_point(x1, x2)
    same, unmatched, epi, con = compare_with_cv2(cv2, x1, x2, A, B, E.reshape(len(x1), 10, 9), n)
    assert same >= 0.99 and unmatched == 0 and epi < 1e-9 and con < 1e-9, (same, unmatched, epi, con)


@pytest.mark.parametrize("p", [0, 7, 12, 20])
def test_counts_selection_and_mask_match_the_oracle(ctx, cfg1, p):
    a, b = _pair(cfg1, p)
    E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a, b)
    samples, nsol, counts = ctx.essential_last_trace()
    assert s["found"] and s["n_samples"] == 1000 and len(samples) == 1000 and s["n_hypotheses"] == nsol.sum()
    # the solutions of the traced samples (same solver, same normalised inputs) scored by the restatement
    x1 = ((a[samples].astype(np.float64) - [CX, CY]) / F); x2 = ((b[samples].astype(np.float64) - [CX, CY]) / F)
    Es, ns = ctx.five_point(x1, x2)
    np.testing.assert_array_equal(ns, nsol)
    hyps = np.concatenate([Es[k, :ns[k]].reshape(-1, 9) for k in range(len(ns))])
    oc, _, _ = ro.score(1, a, b, hyps, AUX, 1.0 / F)
    np.testing.assert_array_equal(counts, oc)
    best, good, it = eo.sequential_select(nsol, counts, len(a))
    assert best >= 0 and good == s["n_inliers"] and it == s["iterations"]
    np.testing.assert_array_equal(E.reshape(-1), hyps[best])
    _, _, om = ro.score(1, a, b, E.reshape(1, 9), AUX, 1.0 / F)
    np.testing.assert_array_equal(inl, om)


def _near_threshold(E, R, t, a, b, mask, dist=50.0):
    """points whose depth in either camera lies within 1e-9 (relative) of 0 or dist: their test may round either way"""
    x1 = (a.astype(np.float64) - [CX, CY]) / F; x2 = (b.astype(np.float64) - [CX, CY]) / F
    Q = cv2.triangulatePoints(np.eye(3, 4), np.c_[R, t], x1.T, x2.T)
    z1 = Q[2] / Q[3]; z2 = (np.c_[R, t] @ (Q / Q[3]))[2]
    near = lambda z: (np.abs(z) < 1e-9 * dist) | (np.abs(z - dist) < 1e-9 * dist)
    return near(z1) | near(z2)


def test_pose_matches_cv2_recover_pose_on_every_pair(ctx, cfg1):
    for p in range(len(cfg1.pairs)):
        a, b = _pair(cfg1, p)
        E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a, b)
        assert s["found"]
        n, Rc, tc, mc = cv2.recoverPose(E, a.astype(np.float64), b.astype(np.float64), focal=F, pp=(CX, CY), mask=inl.reshape(-1, 1).copy())
        np.testing.assert_allclose(R, Rc, rtol=0, atol=1e-9, err_msg=f"pair {p}")
        np.testing.assert_allclose(t, tc.ravel(), rtol=0, atol=1e-9, err_msg=f"pair {p}")
        diff = (pm != 0) != (mc.ravel() != 0)
        assert not np.any(diff & ~_near_threshold(E, R, t, a, b, inl)), (p, np.flatnonzero(diff))
        assert s["n_good"] == int(pm.sum())


def test_pose_matches_cv2_on_synthetic_scenes(ctx):
    for seed in range(6):
        a, b, Rt, tt, _ = synthetic_scene(seed, 800, noise_px=0.5, outliers=0.3)
        E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a, b, seed=seed)
        n, Rc, tc, mc = cv2.recoverPose(E, a.astype(np.float64), b.astype(np.float64), focal=F, pp=(CX, CY), mask=inl.reshape(-1, 1).copy())
        np.testing.assert_allclose(R, Rc, rtol=0, atol=1e-9); np.testing.assert_allclose(t, tc.ravel(), rtol=0, atol=1e-9)
        diff = (pm != 0) != (mc.ravel() != 0)
        assert not np.any(diff & ~_near_threshold(E, R, t, a, b, inl))
        # against the truth: rotation to 0.1 degree, translation direction to 1 degree
        assert _angle(R, Rt) < 0.1, _angle(R, Rt)
        assert np.degrees(np.arccos(np.clip(t @ tt, -1, 1))) < 1.0


def test_against_cv2_statistically(ctx, cfg1):
    """One RANSAC run of either library is one draw: its samples come from its own generator.  Over eight seeds, on every pair:
    the median inlier count is within 10 % of cv2's (single runs spread over 0.87-1.08 of it); and where cv2's pose keeps at
    least half its inliers, cv2's rotation lies no further from ours (median over the seeds) than our own runs lie from each
    other, plus 3 degrees.  On these narrow-angle pairs the rotation of a minimal-sample RANSAC is poorly determined: our runs
    differ from each other by 6 to 54 degrees, so a single run cannot be held to 3 degrees of cv2's."""
    for p in range(len(cfg1.pairs)):
        a, b = _pair(cfg1, p)
        Ec, mc = cv2.findEssentialMat(a, b, F, (CX, CY), cv2.RANSAC, 0.999, 1.0)
        n, Rc, tc, mc2 = cv2.recoverPose(Ec[:3], a, b, focal=F, pp=(CX, CY), mask=mc.copy())
        runs = [ctx.find_camera_matrices(K, a, b, seed=sd) for sd in range(8)]
        counts = [r[5]["n_inliers"] for r in runs]
        assert np.median(counts) >= 0.9 * int(mc.sum()), (p, counts, int(mc.sum()))
        if mc2.sum() >= 0.5 * mc.sum():
            Rs = [r[1] for r in runs]
            spread = max(_angle(A, B) for A in Rs for B in Rs)
            to_cv2 = np.median([_angle(R, Rc) for R in Rs])
            assert to_cv2 <= spread + 3.0, (p, to_cv2, spread)


def test_same_seed_same_bits_and_seed_changes_samples(ctx, cfg1):
    a, b = _pair(cfg1, 3)
    r1 = ctx.find_camera_matrices(K, a, b, seed=11); t1 = ctx.essential_last_trace()
    r2 = ctx.find_camera_matrices(K, a, b, seed=11); t2 = ctx.essential_last_trace()
    for x, y in zip(r1[:5] + t1, r2[:5] + t2):
        np.testing.assert_array_equal(x, y)
    assert r1[5] == r2[5]
    ctx.find_camera_matrices(K, a, b, seed=12)
    assert not np.array_equal(ctx.essential_last_trace()[0], t1[0])


def test_edge_cases(ctx):
    a, b, *_ = synthetic_scene(3, 40)
    for m in (0, 1, 4):                                           # too few correspondences: OK, nothing found
        E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a[:m], b[:m])
        assert s["found"] == 0 and not E.any() and not inl.any()
    E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a[:5], b[:5])   # one sample, the same selection
    assert s["n_samples"] == 1 and s["found"] == 1 and s["n_inliers"] == 5 and s["iterations"] == 1
    same = np.tile(a[:1], (30, 1))                                # all points identical: rank-deficient samples
    E, R, t, inl, pm, s = ctx.find_camera_matrices(K, same, same)
    assert s["found"] == 0 and s["n_hypotheses"] == 0 and np.all(np.isfinite(E))
    with pytest.raises(capi.SfmB200Error, match="outside"):
        ctx.find_camera_matrices(K, a, b, np.arange(10), np.r_[np.arange(9), 40])
    with pytest.raises(capi.SfmB200Error, match="options"):
        ctx.find_camera_matrices(K, a, b, confidence=1.0)
    E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a, b)     # the context still works
    assert s["found"] == 1


def test_whole_replay_with_the_device_stage(ctx, cfg1):
    sfm = runsfm.SfM(cfg1.features, cfg1.size,
                     matchAllPairs=lambda f, pr: stages.matchAllPairs(f, pr, ctx=ctx), matchFeatures=lambda a, b: stages.matchFeatures(a, b, ctx=ctx),
                     triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx), adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx),
                     findHomographyInliers=lambda *a: ransac.findHomographyInliers(*a, ctx=ctx),
                     findCameraMatricesFromMatch=lambda *a: ransac.findCameraMatricesFromMatch_gpu(*a, ctx=ctx),
                     findCameraPoseFrom2D3DMatch=lambda *a: ransac.findCameraPoseFrom2D3DMatch(*a, ctx=ctx))
    sfm.runSfM()
    assert len(sfm.mDoneViews) == 7
    assert 0.5 * len(cfg1.g["final_cloud"]) < len(sfm.mReconstructionCloud) < 2.0 * len(cfg1.g["final_cloud"])
    assert abs(float(sfm.mIntrinsics.K[0, 0]) - float(cfg1.g["final_K"][0, 0])) < 0.15 * float(cfg1.g["final_K"][0, 0])
