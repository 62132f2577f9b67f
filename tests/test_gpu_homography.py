"""Homography RANSAC on the device (sfmb200_find_homography_pairs, SfMStereoUtilities.cpp:51-72): counts and masks identical to
cv2.findHomography(RANSAC, 10) on every crazyhorse pair and on synthetic scenes, H to rounding, the visited samples and their
counts identical to the restatement's, batching and repetition invariance, and the runSfM replay with the batched stage."""
import numpy as np
import pytest

from cfg1_util import Cfg1
import homography_oracle as ho
from homography_util import crazyhorse_pairs, planar_scene, synthetic_scenes
from oracle import cv2_stages
from sfm_toy_library_b200 import capi, ransac, runsfm, stages

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
DEGENERATE = ("collinear", "n4_collinear")       # H is not unique there; counts and masks still are


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _batch(ctx, pairs_ab, **kw):
    """Each (a, b) as its own two images, all pairs in one call."""
    pts = [x for a, b in pairs_ab for x in (a, b)]
    pairs = [(2 * k, 2 * k + 1) for k in range(len(pairs_ab))]
    mq, mt, off = capi.flatten_matches([np.arange(len(a)) for a, _ in pairs_ab], [np.arange(len(b)) for _, b in pairs_ab])
    return ctx.find_homography_pairs(pts, pairs, mq, mt, off, **kw), off


def _check_against_cv2(ctx, names, pairs_ab, off, H, mask, s):
    for k, (name, (a, b)) in enumerate(zip(names, pairs_ab)):
        m = mask[off[k]:off[k + 1]]
        Hc, mc = cv2.findHomography(a, b, cv2.RANSAC, 10.0) if len(a) >= 4 else (None, None)
        if Hc is None:
            assert s["found"][k] == 0 and s["n_inliers"][k] == 0 and not m.any(), name
            continue
        assert s["found"][k] == 1, name
        assert s["n_inliers"][k] == int(mc.sum()) and np.array_equal(m, mc.ravel()), name
        if name not in DEGENERATE:
            assert np.abs(H[k] - Hc).max() <= 1e-6 * np.abs(Hc).max(), (name, np.abs(H[k] - Hc).max())
        o = ho.find_homography(a, b)
        assert s["ransac_inliers"][k] == o["ransac_inliers"] and s["iterations"][k] == o["iterations"], name
        if len(a) > 4:
            q, c = ctx.homography_last_trace(k)
            assert np.array_equal(q, np.array([v[0] for v in o["visited"]]).reshape(-1, 4)), name
            assert np.array_equal(c, np.array([v[1] for v in o["visited"]])), name


def test_crazyhorse_batched_equals_cv2(ctx):
    ab = crazyhorse_pairs(Cfg1())
    (H, mask, s), off = _batch(ctx, ab, record_trace=1)
    _check_against_cv2(ctx, [f"pair{p}" for p in range(len(ab))], ab, off, H, mask, s)


def test_synthetic_and_edge_cases_equal_cv2(ctx):
    sc = synthetic_scenes()
    big = planar_scene(77, 20000, 0.5)
    tiny = planar_scene(78, 3, 0.0)
    names = [n for n, _, _ in sc] + ["empty", "n3", "big20000"]
    ab = [(a, b) for _, a, b in sc] + [(np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32)), tiny, big]
    (H, mask, s), off = _batch(ctx, ab, record_trace=1)
    _check_against_cv2(ctx, names, ab, off, H, mask, s)


def test_single_and_batched_calls_are_identical(ctx):
    ab = crazyhorse_pairs(Cfg1())[:8] + [(a, b) for _, a, b in synthetic_scenes()[8:12]]
    (H, mask, s), off = _batch(ctx, ab)
    (H2, mask2, s2), _ = _batch(ctx, ab)
    assert np.array_equal(H, H2) and np.array_equal(mask, mask2) and all(np.array_equal(s[k], s2[k]) for k in s)
    for k, (a, b) in enumerate(ab):
        (h1, m1, s1), _ = _batch(ctx, [(a, b)])
        assert np.array_equal(h1[0], H[k]) and np.array_equal(m1, mask[off[k]:off[k + 1]])
        assert all(s1[f][0] == s[f][k] for f in s)


def test_indexed_points_and_validation(ctx):
    cfg = Cfg1()
    pairs = cfg.pairs
    mq, mt, off = capi.flatten_matches([m[0] for m in cfg.matches], [m[1] for m in cfg.matches])
    H, mask, s = ctx.find_homography_pairs([f.points for f in cfg.features], pairs, mq, mt, off)
    for p, (a, b) in enumerate(crazyhorse_pairs(cfg)):
        _, mc = cv2.findHomography(a, b, cv2.RANSAC, 10.0)
        assert np.array_equal(mask[off[p]:off[p + 1]], mc.ravel())
    m = np.zeros(len(cfg.matches[0][0]), stages.DMATCH); m["queryIdx"], m["trainIdx"], _ = cfg.matches[0]
    i, j = pairs[0]
    assert ransac.findHomographyInliers_gpu(cfg.features[i], cfg.features[j], m, ctx=ctx) == runsfm.findHomographyInliers_cv2(cfg.features[i], cfg.features[j], m)
    assert ransac.findHomographyInliers_gpu(cfg.features[i], cfg.features[j], m[:3], ctx=ctx) == 0
    bad = mq.copy(); bad[5] = 10 ** 6
    with pytest.raises(capi.SfmB200Error, match="outside"):
        ctx.find_homography_pairs([f.points for f in cfg.features], pairs, bad, mt, off)
    with pytest.raises(capi.SfmB200Error, match="outside"):
        ctx.find_homography_pairs([f.points for f in cfg.features], [(0, 9)] + pairs[1:], mq, mt, off)
    with pytest.raises(capi.SfmB200Error, match="options"):
        ctx.find_homography_pairs([f.points for f in cfg.features], pairs, mq, mt, off, confidence=1.0)
    H2, mask2, s2 = ctx.find_homography_pairs([f.points for f in cfg.features], pairs, mq, mt, off)      # the context still works
    assert np.array_equal(mask, mask2)


def _same(x, y):
    """Equal structure and values; wall-clock fields (`*_time_s` of a bundle adjustment summary) are not compared."""
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x if not str(k).endswith("time_s"))
    if isinstance(x, (list, tuple)):
        return len(x) == len(y) and all(_same(u, v) for u, v in zip(x, y))
    return np.array_equal(np.asarray(x), np.asarray(y))


def test_replay_with_the_batched_stage_equals_the_cv2_replay(ctx):
    cfg = Cfg1()
    common = dict(matchFeatures=cv2_stages.matchFeatures, triangulateViews=cv2_stages.triangulateViews, adjustBundle=cv2_stages.adjustBundle)
    t_cv, t_gpu = [], []
    ref = runsfm.SfM(cfg.features, cfg.size, trace=t_cv, **common)
    ref.createFeatureMatchMatrix()
    order_cv = ref.sortViewsForBaseline()
    gpu = runsfm.SfM(cfg.features, cfg.size, trace=t_gpu,
                     homographyInliersAllPairs=lambda f, pr, m: ransac.homographyInliersAllPairs(f, pr, m, ctx=ctx), **common)
    gpu.createFeatureMatchMatrix()
    order_gpu = gpu.sortViewsForBaseline()
    assert order_gpu == order_cv
    assert gpu.calls["homography"] == 1
    t_cv.clear(); t_gpu.clear()
    ref = runsfm.SfM(cfg.features, cfg.size, trace=t_cv, **common)
    ref.runSfM()
    gpu = runsfm.SfM(cfg.features, cfg.size, trace=t_gpu,
                     homographyInliersAllPairs=lambda f, pr, m: ransac.homographyInliersAllPairs(f, pr, m, ctx=ctx), **common)
    gpu.runSfM()
    assert len(t_gpu) == len(t_cv) and [e["stage"] for e in t_gpu] == [e["stage"] for e in t_cv]
    for x, y in zip(t_gpu, t_cv):
        assert _same(x, y), x["stage"]
