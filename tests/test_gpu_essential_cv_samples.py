"""Essential-matrix RANSAC with cv::findEssentialMat's own samples (sfmb200_essential_options.sampler = SFMB200_SAMPLER_OPENCV):
on every crazyhorse pair and on synthetic scenes (m = 5 and 6, 0-70 % outliers) the traced samples and the iteration count are
the Python replay's (tests/essential_cv_replay.py, pinned to cv2 by test_essential_cv_replay_cpu.py), E is cv2's to 1e-9, the
inlier mask is cv2's mask, and R, t and the pose mask are cv2.recoverPose's on cv2's E and mask.  The pairs call equals its single
calls bit for bit across a hypothesis-group boundary, the seed is ignored, the C++ shim built with SFMB200_SHIM_ESSENTIAL_OPENCV
returns cv2's pruned matches, and in a runSfM replay every findCameraMatricesFromMatch call prunes as cv2 does."""
import os
import subprocess

import numpy as np
import pytest

from cfg1_util import Cfg1
from essential_cv_replay import cv_samples, replay, synthetic_cases
from essential_util import CX, CY, F, canon, synthetic_scene
from sfm_toy_library_b200 import capi, ransac, runsfm, stages

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1]], np.float32)
CV = dict(sampler=capi.SAMPLER_OPENCV)


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


def _sampson(E, a, b):
    E = np.asarray(E, np.float64).reshape(3, 3)
    x1 = np.c_[(a.astype(np.float64) - [CX, CY]) / F, np.ones(len(a))]; x2 = np.c_[(b.astype(np.float64) - [CX, CY]) / F, np.ones(len(b))]
    Ex1 = x1 @ E.T; Etx2 = x2 @ E
    return np.einsum("ij,ij->i", x2, Ex1) ** 2 / (Ex1[:, 0] ** 2 + Ex1[:, 1] ** 2 + Etx2[:, 0] ** 2 + Etx2[:, 1] ** 2)


def _near_depth(R, t, a, b, dist=50.0):
    """points whose depth in either camera lies within 1e-9 (relative) of 0 or dist: their cheirality test may round either way"""
    x1 = (a.astype(np.float64) - [CX, CY]) / F; x2 = (b.astype(np.float64) - [CX, CY]) / F
    Q = cv2.triangulatePoints(np.eye(3, 4), np.c_[R, t], x1.T, x2.T)
    z1 = Q[2] / Q[3]; z2 = (np.c_[R, t] @ (Q / Q[3]))[2]
    near = lambda z: (np.abs(z) < 1e-9 * dist) | (np.abs(z - dist) < 1e-9 * dist)
    return near(z1) | near(z2)


def _check_against_cv2(ctx, a, b, label, exact_masks, e_tol=1e-9):
    """one call under the OpenCV sampler against the replay and cv2; returns (the number of inlier-mask entries that differ from
    cv2's, all within rounding of the threshold, and the largest difference of the normalised E)"""
    E, R, t, inl, pm, s = ctx.find_camera_matrices(K, a, b, **CV)
    smp, nsol, counts = ctx.essential_last_trace()
    r = replay(cv2, a, b, F, (CX, CY))
    m = len(a)
    assert s["found"] == 1 and r["best"] >= 0, label
    assert s["n_samples"] == (1 if m == 5 else 1000), (label, s)
    np.testing.assert_array_equal(smp, cv_samples(m, s["n_samples"]), err_msg=label)
    np.testing.assert_array_equal(smp[:r["iterations"]], r["samples"], err_msg=label)
    assert s["iterations"] == r["iterations"], (label, s["iterations"], r["iterations"])
    Ec, mc = cv2.findEssentialMat(a, b, F, (CX, CY), cv2.RANSAC, 0.999, 1.0)
    if m == 5:
        # cv2 stacks every solution of the one sample, each with all five points inlying; the selection keeps the first in the
        # solver's order (ascending root here), one of cv2's, with the five points as inliers
        d = min(np.abs(canon(E) - canon(Ec[3 * k:3 * k + 3])).max() for k in range(Ec.shape[0] // 3))
        assert d < e_tol and inl.all() and s["n_inliers"] == 5, (label, d)
        return 0, d
    Ec = Ec[:3]; mc = mc.ravel()
    d = np.abs(canon(E) - canon(Ec)).max()
    assert d < e_tol, (label, d)
    diff = np.flatnonzero(inl != mc)
    t2 = (1.0 / F) ** 2
    # within rounding of the threshold: on either side of it under one of the two E, or within 1e-6 of it
    e_ours, e_cv = _sampson(E, a, b), _sampson(Ec, a, b)
    near = ((e_ours <= t2) != (e_cv <= t2)) | (np.abs(e_cv - t2) <= 1e-6 * t2)
    if exact_masks:
        assert len(diff) == 0, (label, diff)
    assert np.all(near[diff]), (label, diff)
    assert s["n_inliers"] == int(inl.sum())
    n, Rc, tc, pc = cv2.recoverPose(Ec, a.astype(np.float64), b.astype(np.float64), focal=F, pp=(CX, CY), mask=mc.reshape(-1, 1).astype(np.uint8))
    tol = max(1e-9, 10 * d)                                   # R and t follow E's difference
    np.testing.assert_allclose(R, Rc, rtol=0, atol=tol, err_msg=label)
    np.testing.assert_allclose(t, tc.ravel(), rtol=0, atol=tol, err_msg=label)
    pdiff = (pm != 0) != (pc.ravel() != 0)
    if exact_masks:
        assert not pdiff.any(), (label, np.flatnonzero(pdiff))
    assert not np.any(pdiff & ~_near_depth(R, t, a, b) & ~np.isin(np.arange(m), diff)), (label, np.flatnonzero(pdiff))
    return len(diff), d


def test_crazyhorse_pairs_are_cv2s(ctx, cfg1):
    worst = 0.0
    for p in range(len(cfg1.pairs)):
        a, b = _pair(cfg1, p)
        worst = max(worst, _check_against_cv2(ctx, a, b, f"pair {p}", exact_masks=True)[1])
    print("crazyhorse: largest difference of the normalised E from cv2's:", worst)


def test_synthetic_scenes_are_cv2s(ctx):
    """E to 1e-6: where the winning sample is ill-conditioned the two five-point solvers agree only to a few 1e-7 (a 60-match scene
    at 70 % outliers); the masks may then differ at points within rounding of the threshold, which are counted."""
    flips, worst = 0, []
    for seed, n, out in synthetic_cases():
        a, b, *_ = synthetic_scene(seed, n, noise_px=0.5, outliers=out)
        k, d = _check_against_cv2(ctx, a, b, f"scene {seed} n {n} outliers {out}", exact_masks=False, e_tol=1e-6)
        flips += k; worst.append(d)
    print("synthetic: inlier-mask entries within rounding of the threshold that differ from cv2's:", flips)
    print("synthetic: difference of the normalised E from cv2's per scene:", ["%.1e" % d for d in worst])


@pytest.mark.parametrize("m", [5, 6, 7, 9])
def test_tiny_sets_are_cv2s(ctx, m):
    a, b, *_ = synthetic_scene(40 + m, m, noise_px=0.5)
    _check_against_cv2(ctx, a, b, f"m {m}", exact_masks=True)


def test_seed_is_ignored(ctx, cfg1):
    a, b = _pair(cfg1, 5)
    r1 = ctx.find_camera_matrices(K, a, b, seed=0, **CV); t1 = ctx.essential_last_trace()
    r2 = ctx.find_camera_matrices(K, a, b, seed=12345, **CV); t2 = ctx.essential_last_trace()
    for x, y in zip(r1[:5] + t1, r2[:5] + t2):
        np.testing.assert_array_equal(x, y)
    assert r1[5] == r2[5]
    seeded = ctx.find_camera_matrices(K, a, b)
    assert not np.array_equal(ctx.essential_last_trace()[0], t1[0]) and seeded[5]["found"]


def test_unknown_sampler_is_refused(ctx, cfg1):
    a, b = _pair(cfg1, 0)
    for bad in (-1, 2):
        with pytest.raises(capi.SfmB200Error, match="sampler"):
            ctx.find_camera_matrices(K, a, b, sampler=bad)
        with pytest.raises(capi.SfmB200Error, match="sampler"):
            ctx.find_camera_matrices_pairs(K, [a, b], [(0, 1)], np.arange(len(a)), np.arange(len(a)), np.array([0, len(a)]), sampler=bad)
    assert ctx.find_camera_matrices(K, a, b, **CV)[5]["found"]


def test_pairs_equal_single_calls_across_a_group_boundary(ctx, cfg1):
    """15 copies of the 21 pairs (315 pairs at 1000 samples) span two groups of the 256 MB hypothesis budget (279 pairs each)."""
    n = len(cfg1.pairs)
    singles = [ctx.find_camera_matrices(K, *_pair(cfg1, p), **CV) for p in range(n)]
    order = [p for _ in range(15) for p in range(n)]
    pts = [f.points for f in cfg1.features]
    mq, mt, off = capi.flatten_matches([cfg1.matches[p][0] for p in order], [cfg1.matches[p][1] for p in order])
    E, R, t, inl, pm, s = ctx.find_camera_matrices_pairs(K, pts, [cfg1.pairs[p] for p in order], mq, mt, off, seed=99, **CV)
    assert len(order) * 1000 > (256 << 20) // 960
    for k, p in enumerate(order):
        sl = slice(int(off[k]), int(off[k + 1]))
        E1, R1, t1, inl1, pm1, s1 = singles[p]
        for x, y, name in ((E[k], E1, "E"), (R[k], R1, "R"), (t[k], t1, "t"), (inl[sl], inl1, "inlier_mask"), (pm[sl], pm1, "pose_mask")):
            np.testing.assert_array_equal(x, y, err_msg=f"batch entry {k} (pair {p}) {name}")
        assert {q: int(v[k]) for q, v in s.items()} == s1, (k, s1)


def _write_pairs(path, cfg1):
    with open(path, "wb") as f:
        f.write(np.int32(len(cfg1.pairs)).tobytes()); f.write(K.astype(np.float32).tobytes())
        for p, (i, j) in enumerate(cfg1.pairs):
            q, t, _ = cfg1.matches[p]
            for pts in (cfg1.features[i].points, cfg1.features[j].points):
                f.write(np.int32(len(pts)).tobytes()); f.write(np.ascontiguousarray(pts, np.float32).tobytes())
            f.write(np.int32(len(q)).tobytes()); f.write(np.asarray(q, np.int32).tobytes()); f.write(np.asarray(t, np.int32).tobytes())


def _read_results(path, n_pairs):
    buf = np.fromfile(path, np.uint8); o = 0; out = []
    take = lambda k, dt: (np.frombuffer(buf[o:o + 4 * k].tobytes(), dt), o + 4 * k)
    for _ in range(n_pairs):
        (ok, n), o = take(2, np.int32)
        q, o = take(int(n), np.int32); t, o = take(int(n), np.int32); P, o = take(12, np.float32)
        out.append((int(ok), q, t, P.reshape(3, 4)))
    assert o == len(buf)
    return out


def test_cpp_shim_gives_cv2s_pruned_matches(cfg1, tmp_path):
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_shim_essential_opencv")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    _write_pairs(tmp_path / "in.bin", cfg1)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "SHIM_ESSENTIAL_OPENCV_TEST DONE" in r.stdout
    for p, (ok, q, t, P) in enumerate(_read_results(tmp_path / "out.bin", len(cfg1.pairs))):
        i, j = cfg1.pairs[p]; mq, mt, _ = cfg1.matches[p]
        m = np.zeros(len(mq), stages.DMATCH); m["queryIdx"] = mq; m["trainIdx"] = mt
        _, pruned, _, Pc = runsfm.findCameraMatricesFromMatch_cv2(stages.Intrinsics(K=K), m, cfg1.features[i], cfg1.features[j])
        assert ok == 1, p
        np.testing.assert_array_equal(q, pruned["queryIdx"], err_msg=f"pair {p}")
        np.testing.assert_array_equal(t, pruned["trainIdx"], err_msg=f"pair {p}")
        np.testing.assert_allclose(P, Pc, rtol=0, atol=1e-6, err_msg=f"pair {p}")


def test_runsfm_replay_prunes_as_cv2_does(ctx, cfg1):
    calls = []

    def device_stage(intrinsics, matches, left, right):
        got = ransac.findCameraMatricesFromMatch_gpu(intrinsics, matches, left, right, ctx=ctx, sampler=capi.SAMPLER_OPENCV)
        try:
            ref = runsfm.findCameraMatricesFromMatch_cv2(intrinsics, matches, left, right)
        except cv2.error:                                     # cv::findEssentialMat asserts below 5 points
            ref = (False, matches[:0], None, None)
        calls.append((len(matches), got, ref))
        return got

    sfm = runsfm.SfM(cfg1.features, cfg1.size,
                     matchAllPairs=lambda f, pr: stages.matchAllPairs(f, pr, ctx=ctx), matchFeatures=lambda a, b: stages.matchFeatures(a, b, ctx=ctx),
                     triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx), adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx),
                     findHomographyInliers=lambda *a: ransac.findHomographyInliers_gpu(*a, ctx=ctx),
                     findCameraMatricesFromMatch=device_stage,
                     findCameraPoseFrom2D3DMatch=lambda *a: ransac.findCameraPoseFrom2D3DMatch(*a, ctx=ctx))
    sfm.runSfM()
    assert len(sfm.mDoneViews) == 7 and len(calls) > 6
    for k, (m, got, ref) in enumerate(calls):
        assert got[0] == ref[0], (k, m)
        np.testing.assert_array_equal(got[1]["queryIdx"], ref[1]["queryIdx"], err_msg=f"call {k}")
        np.testing.assert_array_equal(got[1]["trainIdx"], ref[1]["trainIdx"], err_msg=f"call {k}")
        if got[0]:
            np.testing.assert_allclose(got[3], ref[3], rtol=0, atol=1e-6, err_msg=f"call {k}")
    print("findCameraMatricesFromMatch calls, all pruned as cv2 prunes:", len(calls))
