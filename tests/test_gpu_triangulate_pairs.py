"""Two-view triangulation for many image pairs in one call (sfmb200_triangulate_pairs): every pair's X, keep and n_keep bitwise
equal to the single-pair call, whatever else is in the batch; the crazyhorse calls against their goldens; a 1225-pair synthetic
batch against the oracle; the edge cases; the binding's refusals; and the runSfM replay with the batched stage injected.  The
host-side refusals of the C call are in test_gpu_pair_batch.py."""
import numpy as np
import pytest

from cfg1_util import Cfg1
from sfm_toy_library_b200 import capi, ransac, runsfm, stages, synth

pytestmark = pytest.mark.gpu
REL_TOL = 1e-5        # as tests/test_gpu_triangulate.py
ERR_TOL = 1e-3


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cfg1():
    return Cfg1()


def _assert_equal_to_single_calls(ctx, K, poses, pts, pairs, mq, mt, off, out, which=None):
    X, keep, nk = out
    assert X.shape == (len(mq), 3) and keep.shape == (len(mq),) and nk.shape == (len(pairs),)
    for p in (range(len(pairs)) if which is None else which):
        i, j = pairs[p]
        sl = slice(int(off[p]), int(off[p + 1]))
        X1, keep1, nk1 = ctx.triangulate(K, poses[p][0], poses[p][1], pts[i], pts[j], mq[sl], mt[sl])
        np.testing.assert_array_equal(X[sl], X1, err_msg=f"pair {p} X")
        np.testing.assert_array_equal(keep[sl], keep1, err_msg=f"pair {p} keep")
        assert nk[p] == nk1 == int(keep1.sum()), p


def _cfg1_groups(cfg1):
    """the recorded calls grouped by their K: call 0 is the baseline, every other group one addMoreViews loop"""
    groups = {}
    for k in range(cfg1.n_tri):
        groups.setdefault(cfg1.tri(k)["K"].tobytes(), []).append(k)
    return list(groups.values())


def _cfg1_batch(cfg1, calls, K=None):
    cs = [cfg1.tri(k) for k in calls]
    pairs = [tuple(int(x) for x in c["pair"]) for c in cs]
    poses = [(c["Pl"], c["Pr"]) for c in cs]
    mq, mt, off = capi.flatten_matches([c["mq"] for c in cs], [c["mt"] for c in cs])
    return (cs[0]["K"] if K is None else K), poses, [f.points for f in cfg1.features], pairs, mq, mt, off


def test_crazyhorse_calls_equal_their_single_calls_and_goldens(ctx, cfg1):
    groups = _cfg1_groups(cfg1)
    assert len(groups) == 6 and sum(len(g) for g in groups) == cfg1.n_tri == 21
    n = 0
    for calls in groups:
        for order in (calls, calls[::-1], calls + [calls[0]]):
            K, poses, pts, pairs, mq, mt, off = args = _cfg1_batch(cfg1, order)
            out = ctx.triangulate_pairs(K, poses, pts, pairs, mq, mt, off)
            _assert_equal_to_single_calls(ctx, *args, out)
            X, keep, nk = out
            for p, k in enumerate(order):
                c = cfg1.tri(k)
                sl = slice(int(off[p]), int(off[p + 1]))
                sel = np.nonzero(keep[sl])[0]
                back = np.stack([c["mq"][sel], c["mt"][sel]], 1).reshape(-1, 2)
                np.testing.assert_array_equal(back, c["back"], err_msg=f"call {k}")
                if len(sel):
                    rel = np.linalg.norm(X[sl][sel] - c["X"], axis=1) / np.maximum(np.linalg.norm(c["X"], axis=1), 1e-12)
                    assert rel.max() < REL_TOL, (k, rel.max())
                if order is calls:
                    n += len(sel)
        np.testing.assert_array_equal(out[0][int(off[0]):int(off[1])], out[0][int(off[-2]):])          # the pair that appears twice
    assert n > 3000


def test_all_crazyhorse_calls_in_one_batch(ctx, cfg1):
    """the 21 calls of all loops in one call (with the K of the baseline), forwards and backwards"""
    K = cfg1.tri(0)["K"]
    for order in (list(range(cfg1.n_tri)), list(range(cfg1.n_tri))[::-1]):
        args = _cfg1_batch(cfg1, order, K)
        _assert_equal_to_single_calls(ctx, *args, ctx.triangulate_pairs(*args))


def test_synthetic_1225_pairs(ctx, oracle):
    K, poses, pts, pairs, mq, mt, off = args = synth.make_triangulation_pairs(50, seed=0)
    assert len(pairs) == 1225 and 0.9e6 < off[-1] < 1.1e6
    l0 = ctx.kernel_launches
    X, keep, nk = out = ctx.triangulate_pairs(*args)
    assert ctx.kernel_launches - l0 == int((np.diff(off) > 0).sum())      # the single call's kernel, once per pair
    np.testing.assert_array_equal(nk, np.add.reduceat(keep.astype(np.int64), off[:-1]))
    assert 0.95 < keep.mean() < 0.995
    rs = np.random.RandomState(1)
    _assert_equal_to_single_calls(ctx, *args, out, sorted(set(rs.choice(1225, 24, replace=False)) | {0, 1224}))
    # every pair against the oracle restatement of triangulateViews, within the tolerances of test_gpu_triangulate.py
    Xo = np.empty_like(X); ko = np.empty_like(keep); eo = np.empty((len(keep), 2))
    for p, (i, j) in enumerate(pairs):
        sl = slice(int(off[p]), int(off[p + 1]))
        Xo[sl], ko[sl], eo[sl] = oracle.triangulate(K, poses[p][0], poses[p][1], pts[i], pts[j], mq[sl], mt[sl])
    good = ko.astype(bool)
    rel = np.linalg.norm(X[good] - Xo[good], axis=1) / np.linalg.norm(Xo[good], axis=1)
    assert rel.max() < REL_TOL, rel.max()
    diff = keep != ko
    if diff.any():
        assert (np.abs(np.max(eo[diff], axis=1) - 10.0) < ERR_TOL).all()


def _two_views(cfg1):
    c = cfg1.tri(4)
    i, j = (int(x) for x in c["pair"])
    return c["K"], c["Pl"], c["Pr"], cfg1.features[i].points, cfg1.features[j].points


def test_edge_cases(ctx, cfg1):
    K, Pl, Pr, a, b = _two_views(cfg1)
    na, nb = len(a), len(b)
    rs = np.random.RandomState(3)
    # images: a, b, and a copy of a; matches that touch the first and the last key point of every image
    pts = [a, b, a.copy()]
    ends_a = np.r_[0, na - 1, rs.randint(0, na, 200)]; ends_b = np.r_[0, nb - 1, rs.randint(0, nb, 200)]
    cases = [((0, 1), (np.zeros(0), np.zeros(0))), ((0, 1), (ends_a, ends_b)), ((0, 1), (np.zeros(0), np.zeros(0))),
             ((2, 1), (ends_a[::-1], ends_b[::-1])), ((1, 2), (np.r_[nb - 1, 0], np.r_[na - 1, 0])), ((0, 1), (np.zeros(0), np.zeros(0)))]
    pairs = [c[0] for c in cases]
    poses = [(Pl, Pr)] * len(cases)
    mq, mt, off = capi.flatten_matches([c[1][0] for c in cases], [c[1][1] for c in cases])
    out = ctx.triangulate_pairs(K, poses, pts, pairs, mq, mt, off)
    assert out[2][0] == out[2][2] == out[2][5] == 0
    _assert_equal_to_single_calls(ctx, K, poses, pts, pairs, mq, mt, off, out)
    # only pairs without matches; no pairs at all (n_keep = NULL and the C call without pairs: test_gpu_pair_batch.py)
    X, keep, nk = ctx.triangulate_pairs(K, poses[:2], pts, pairs[:1] * 2, np.zeros(0), np.zeros(0), [0, 0, 0])
    assert X.shape == (0, 3) and keep.shape == (0,) and list(nk) == [0, 0]
    X, keep, nk = ctx.triangulate_pairs(K, np.zeros((0, 2, 3, 4)), pts, np.zeros((0, 2)), np.zeros(0), np.zeros(0), [0])
    assert X.shape == (0, 3) and nk.shape == (0,)


def test_invalid_inputs_are_refused_and_the_context_stays_usable(ctx, cfg1):
    """through the binding: its own shape checks, and a refusal of the C call; the full table of the C call's refusals is in
    test_gpu_pair_batch.py"""
    K, Pl, Pr, a, b = _two_views(cfg1)
    idx = np.arange(60)
    good = dict(K=K, poses=[(Pl, Pr)], points=[a, b], pairs=[(0, 1)], match_q=idx, match_t=idx, match_off=[0, 60])
    ref = ctx.triangulate_pairs(**good)
    X1, keep1, nk1 = ctx.triangulate(K, Pl, Pr, a, b, idx, idx)
    np.testing.assert_array_equal(ref[0], X1); np.testing.assert_array_equal(ref[1], keep1); assert ref[2][0] == nk1
    bad = [(dict(poses=[(Pl, Pr)] * 2), ValueError, "one \\(Pleft, Pright\\) per pair"),
           (dict(match_off=[0, 59]), ValueError, "match_off must have"),
           (dict(pairs=[(0, 2)]), capi.SfmB200Error, "outside \\[0, 2\\)"),
           (dict(match_q=np.r_[idx[:59], len(a)]), capi.SfmB200Error, "indexes outside its images")]
    for change, err, msg in bad:
        with pytest.raises(err, match=msg):
            ctx.triangulate_pairs(**{**good, **change})
        for x, y in zip(ctx.triangulate_pairs(**good), ref):
            np.testing.assert_array_equal(x, y)


def _assert_same(x, y, where):
    if isinstance(x, dict):
        assert isinstance(y, dict) and x.keys() == y.keys(), where
        for k in x:
            if "time" not in k and not k.endswith("_ms_total"):      # wall-clock fields of a solver summary
                _assert_same(x[k], y[k], f"{where}.{k}")
    elif isinstance(x, (list, tuple)) and not (x and isinstance(x[0], (int, np.integer))):
        assert isinstance(y, (list, tuple)) and len(x) == len(y), where
        for k, (a, b) in enumerate(zip(x, y)):
            _assert_same(a, b, f"{where}[{k}]")
    else:
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y), err_msg=where)


def _replay(ctx, cfg1, batched):
    kw = dict(matchAllPairs=lambda f, pr: stages.matchAllPairs(f, pr, ctx=ctx), matchFeatures=lambda a, b: stages.matchFeatures(a, b, ctx=ctx),
              triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx), adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx),
              findHomographyInliers=lambda *a: ransac.findHomographyInliers(*a, ctx=ctx),
              findCameraPoseFrom2D3DMatch=lambda *a: ransac.findCameraPoseFrom2D3DMatch(*a, ctx=ctx),
              findCameraMatricesManyPairs=lambda intr, f, pr, m: ransac.cameraMatricesManyPairs(intr, f, pr, m, ctx=ctx))
    if batched:
        kw["triangulateManyPairs"] = lambda *a: stages.triangulateManyPairs(*a, ctx=ctx)
    trace = []
    sfm = runsfm.SfM(cfg1.features, cfg1.size, trace=trace, **kw)
    sfm.runSfM()
    return sfm, trace


def test_replay_with_the_batched_stage(ctx, cfg1):
    seq, seq_trace = _replay(ctx, cfg1, False)
    bat, bat_trace = _replay(ctx, cfg1, True)
    assert len(bat.mDoneViews) == 7
    added = sum(1 for e in bat_trace if e["stage"] == "pnp" and e["ok"])
    n_tri = sum(1 for e in bat_trace if e["stage"] == "triangulate")
    assert bat.calls["triangulate"] == 1 + added and seq.calls["triangulate"] == n_tri > bat.calls["triangulate"]
    _assert_same(seq_trace, bat_trace, "trace")
    np.testing.assert_array_equal(np.array([p.p for p in seq.mReconstructionCloud]), np.array([p.p for p in bat.mReconstructionCloud]))
    assert [p.originatingViews for p in seq.mReconstructionCloud] == [p.originatingViews for p in bat.mReconstructionCloud]
    np.testing.assert_array_equal(np.array(seq.mCameraPoses), np.array(bat.mCameraPoses))
    np.testing.assert_array_equal(seq.mIntrinsics.K, bat.mIntrinsics.K)
    for l in range(seq.n):
        for r in range(seq.n):
            np.testing.assert_array_equal(seq.mFeatureMatchMatrix[l][r], bat.mFeatureMatchMatrix[l][r], err_msg=f"matches {l},{r}")
