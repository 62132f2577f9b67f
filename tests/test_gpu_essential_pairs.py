"""Essential-matrix RANSAC and pose recovery for many image pairs in one call (sfmb200_find_camera_matrices_pairs): every pair's
outputs bitwise equal to the single-pair call, whatever else is in the batch; the per-pair edge cases; a batch larger than one group
of the hypothesis budget; the refusals of options and K; and the runSfM replay with the batched stage injected.  The host-side
refusals of the batch layout are in test_gpu_pair_batch.py."""
import numpy as np
import pytest

from cfg1_util import Cfg1
from essential_util import CX, CY, F, synthetic_scene
from sfm_toy_library_b200 import capi, ransac, runsfm, stages

pytestmark = pytest.mark.gpu
K = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1]], np.float32)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cfg1():
    return Cfg1()


def _crazyhorse(cfg1, order):
    pts = [f.points for f in cfg1.features]
    pairs = [cfg1.pairs[p] for p in order]
    mq, mt, off = capi.flatten_matches([cfg1.matches[p][0] for p in order], [cfg1.matches[p][1] for p in order])
    return pts, pairs, mq, mt, off


def _assert_equal_to_single_calls(ctx, pts, pairs, mq, mt, off, out, which=None, **kw):
    E, R, t, inl, pm, s = out
    for p in (range(len(pairs)) if which is None else which):
        i, j = pairs[p]
        sl = slice(int(off[p]), int(off[p + 1]))
        E1, R1, t1, inl1, pm1, s1 = ctx.find_camera_matrices(K, pts[i], pts[j], mq[sl], mt[sl], **kw)
        for x, y, name in ((E[p], E1, "E"), (R[p], R1, "R"), (t[p], t1, "t"), (inl[sl], inl1, "inlier_mask"), (pm[sl], pm1, "pose_mask")):
            np.testing.assert_array_equal(x, y, err_msg=f"pair {p} {name}")
        assert {k: int(v[p]) for k, v in s.items()} == s1, (p, s1)


@pytest.mark.parametrize("seed", [0, 7])
def test_crazyhorse_pairs_equal_their_single_calls(ctx, cfg1, seed):
    n = len(cfg1.pairs)
    for order in (list(range(n)), list(range(n))[::-1], list(range(n)) + [4]):
        args = _crazyhorse(cfg1, order)
        out = ctx.find_camera_matrices_pairs(K, *args, seed=seed)
        assert out[5]["found"].all() and (out[5]["n_samples"] == 1000).all()
        _assert_equal_to_single_calls(ctx, *args, out, seed=seed)
    np.testing.assert_array_equal(out[0][4], out[0][-1])            # the pair that appears twice


def test_mixed_batch(ctx):
    a, b, *_ = synthetic_scene(3, 300, noise_px=0.5, outliers=0.3)
    same = np.tile(a[:1], (30, 1))
    pts = [a, b, same, same.copy()]
    ident = lambda m: (np.arange(m), np.arange(m))
    cases = [((0, 1), ident(0)), ((0, 1), ident(300)), ((0, 1), ident(1)), ((2, 3), ident(30)), ((0, 1), ident(4)),
             ((0, 1), ident(5)), ((1, 0), ident(200)), ((0, 1), ident(0))]
    pairs = [c[0] for c in cases]
    mq, mt, off = capi.flatten_matches([c[1][0] for c in cases], [c[1][1] for c in cases])
    out = ctx.find_camera_matrices_pairs(K, pts, pairs, mq, mt, off)
    s = out[5]
    np.testing.assert_array_equal(s["found"], [0, 1, 0, 0, 0, 1, 1, 0])
    np.testing.assert_array_equal(s["n_samples"], [0, 1000, 0, 1000, 0, 1, 1000, 0])
    assert s["n_hypotheses"][3] == 0 and s["n_inliers"][5] == 5 and s["iterations"][5] == 1
    assert all(np.all(np.isfinite(x)) for x in out[:3])
    _assert_equal_to_single_calls(ctx, pts, pairs, mq, mt, off, out)


def _angle(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


def test_batch_larger_than_one_hypothesis_group(ctx):
    """300 pairs at max_iters 1000 hold 288 MB of hypotheses: two groups of the 256 MB budget (279 pairs fit in one)."""
    rs = np.random.RandomState(11)
    pts, pairs, qs, truth = [], [], [], []
    for k in range(300):
        a, b, Rt, tt, _ = synthetic_scene(1000 + k, int(rs.randint(800, 1201)), noise_px=0.5, outliers=0.3)
        pts += [a, b]; pairs.append((2 * k, 2 * k + 1)); qs.append(np.arange(len(a))); truth.append((Rt, tt))
    mq, mt, off = capi.flatten_matches(qs, qs)
    l0 = ctx.kernel_launches
    out = ctx.find_camera_matrices_pairs(K, pts, pairs, mq, mt, off, seed=3)
    assert ctx.kernel_launches - l0 == 2 * 3 + 2             # solve, score, select per group; cheirality and pose once
    E, R, t, inl, pm, s = out
    assert s["found"].all()
    rot = [_angle(R[p], truth[p][0]) for p in range(300)]
    tra = [np.degrees(np.arccos(np.clip(t[p] @ truth[p][1], -1, 1))) for p in range(300)]
    assert max(rot) < 0.1 and max(tra) < 1.0, (max(rot), max(tra))
    which = sorted(set(rs.choice(300, 16, replace=False)) | {0, 278, 279, 299})    # both sides of the group boundary
    _assert_equal_to_single_calls(ctx, pts, pairs, mq, mt, off, out, which, seed=3)


def test_invalid_inputs_are_refused_and_the_context_stays_usable(ctx):
    """the options and K of the single call; the refusals of the batch layout are in test_gpu_pair_batch.py"""
    a, b, *_ = synthetic_scene(5, 60)
    idx = np.arange(60)
    good = ([a, b], [(0, 1)], idx, idx, [0, 60])
    assert ctx.find_camera_matrices_pairs(K, *good)[5]["found"][0] == 1
    bad = [(K, dict(confidence=1.0), "essential options"),
           (K, dict(max_iters=0), "essential options"),
           (np.zeros((3, 3)), {}, "focal length")]
    for K_, kw, msg in bad:
        with pytest.raises(capi.SfmB200Error, match=msg):
            ctx.find_camera_matrices_pairs(K_, *good, **kw)
        assert ctx.find_camera_matrices_pairs(K, *good)[5]["found"][0] == 1
    E, R, t, inl, pm, s = ctx.find_camera_matrices_pairs(K, [a, b], np.zeros((0, 2)), np.zeros(0), np.zeros(0), [0])
    assert E.shape == (0, 3, 3) and len(s["found"]) == 0


def test_trace_hook_after_batched_calls(ctx, cfg1):
    args = _crazyhorse(cfg1, [2])
    ctx.find_camera_matrices_pairs(K, *args)
    assert len(ctx.essential_last_trace()[0]) == 1000
    ctx.find_camera_matrices_pairs(K, *_crazyhorse(cfg1, [2, 3]))
    assert len(ctx.essential_last_trace()[0]) == 0


def _replay(ctx, cfg1, batched):
    kw = dict(matchAllPairs=lambda f, pr: stages.matchAllPairs(f, pr, ctx=ctx), matchFeatures=lambda a, b: stages.matchFeatures(a, b, ctx=ctx),
              triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx), adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx),
              findHomographyInliers=lambda *a: ransac.findHomographyInliers(*a, ctx=ctx),
              findCameraPoseFrom2D3DMatch=lambda *a: ransac.findCameraPoseFrom2D3DMatch(*a, ctx=ctx))
    if batched:
        kw["findCameraMatricesManyPairs"] = lambda intr, f, pr, m: ransac.cameraMatricesManyPairs(intr, f, pr, m, ctx=ctx)
    else:
        kw["findCameraMatricesFromMatch"] = lambda *a: ransac.findCameraMatricesFromMatch_gpu(*a, ctx=ctx)
    trace = []
    sfm = runsfm.SfM(cfg1.features, cfg1.size, trace=trace, **kw)
    sfm.runSfM()
    return sfm, trace


def test_replay_with_the_batched_stage(ctx, cfg1):
    seq, _ = _replay(ctx, cfg1, False)
    bat, trace = _replay(ctx, cfg1, True)
    assert len(bat.mDoneViews) == 7
    added = sum(1 for e in trace if e["stage"] == "pnp" and e["ok"])
    assert bat.calls["essential"] == 1 + added == 6 and seq.calls["essential"] > 6
    np.testing.assert_array_equal(np.array([p.p for p in seq.mReconstructionCloud]), np.array([p.p for p in bat.mReconstructionCloud]))
    np.testing.assert_array_equal(np.array(seq.mCameraPoses), np.array(bat.mCameraPoses))
    np.testing.assert_array_equal(seq.mIntrinsics.K, bat.mIntrinsics.K)
