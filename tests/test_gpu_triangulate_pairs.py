"""Two-view triangulation for many image pairs in one call (sfmb200_triangulate_pairs): every pair's X, keep and n_keep bitwise
equal to the single-pair call, whatever else is in the batch; the crazyhorse calls against their goldens; a 1225-pair synthetic
batch against the oracle; the edge cases; the host-side refusals; and the runSfM replay with the batched stage injected."""
import ctypes as C

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


def _flatten(q_list, t_list):
    off = np.zeros(len(q_list) + 1, np.int64); off[1:] = np.cumsum([len(q) for q in q_list])
    cat = lambda xs: np.concatenate([np.asarray(x, np.int32) for x in xs]) if xs else np.zeros(0, np.int32)
    return cat(q_list), cat(t_list), off


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
    mq, mt, off = _flatten([c["mq"] for c in cs], [c["mt"] for c in cs])
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


def _raw(ctx, K, poses, pts, img_off, pairs, mq, mt, moff, with_nkeep=True):
    """the C call with the caller's own offsets (the binding derives img_off itself); returns (X, keep, n_keep or None)"""
    allp = np.ascontiguousarray(np.concatenate(pts), np.float32); img_off = np.asarray(img_off, np.int32)
    pairs = np.asarray(pairs, np.int32).reshape(-1, 2); mq = np.asarray(mq, np.int32); mt = np.asarray(mt, np.int32)
    moff = np.asarray(moff, np.int64); Kf = np.ascontiguousarray(K, np.float32).reshape(9)
    poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 24)
    P = len(pairs); M = max(len(mq), 1)
    X = np.full((M, 3), np.nan, np.float32); keep = np.full(M, 7, np.uint8); nk = np.full(max(P, 1), -1, np.int32)
    ptr = lambda x, tp: x.ctypes.data_as(C.POINTER(tp))
    ctx._check(capi.lib().sfmb200_triangulate_pairs(ctx._h, ptr(Kf, C.c_float), ptr(poses, C.c_float), ptr(allp, C.c_float), ptr(img_off, C.c_int32),
                                                    len(img_off) - 1, ptr(pairs, C.c_int32), P, ptr(mq, C.c_int32), ptr(mt, C.c_int32),
                                                    ptr(moff, C.c_int64), C.c_float(10.0), ptr(X, C.c_float), ptr(keep, C.c_uint8),
                                                    ptr(nk, C.c_int32) if with_nkeep else None))
    return X[:len(mq)], keep[:len(mq)], (nk[:P] if with_nkeep else None)


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
    mq, mt, off = _flatten([c[1][0] for c in cases], [c[1][1] for c in cases])
    out = ctx.triangulate_pairs(K, poses, pts, pairs, mq, mt, off)
    assert out[2][0] == out[2][2] == out[2][5] == 0
    _assert_equal_to_single_calls(ctx, K, poses, pts, pairs, mq, mt, off, out)
    # n_keep = NULL: the same X and keep
    img_off = np.r_[0, np.cumsum([len(p) for p in pts])]
    X, keep, nk = _raw(ctx, K, np.stack([np.stack(p) for p in poses]), pts, img_off, pairs, mq, mt, off, with_nkeep=False)
    assert nk is None
    np.testing.assert_array_equal(X, out[0]); np.testing.assert_array_equal(keep, out[1])
    # only pairs without matches; no pairs at all
    X, keep, nk = ctx.triangulate_pairs(K, poses[:2], pts, pairs[:1] * 2, np.zeros(0), np.zeros(0), [0, 0, 0])
    assert X.shape == (0, 3) and keep.shape == (0,) and list(nk) == [0, 0]
    X, keep, nk = ctx.triangulate_pairs(K, np.zeros((0, 2, 3, 4)), pts, np.zeros((0, 2)), np.zeros(0), np.zeros(0), [0])
    assert X.shape == (0, 3) and nk.shape == (0,)
    _, _, nk = _raw(ctx, K, np.zeros((0, 24)), pts, img_off, np.zeros((0, 2)), np.zeros(0), np.zeros(0), [0])
    assert nk.shape == (0,)


def test_invalid_inputs_are_refused_and_the_context_stays_usable(ctx, cfg1):
    K, Pl, Pr, a, b = _two_views(cfg1)
    idx = np.arange(60)
    pose = np.stack([Pl, Pr]).reshape(1, 24)
    good = dict(img_off=[0, len(a), len(a) + len(b)], pairs=[(0, 1)], mq=idx, mt=idx, moff=[0, 60])
    ref = _raw(ctx, K, pose, [a, b], **good)
    X1, keep1, nk1 = ctx.triangulate(K, Pl, Pr, a, b, idx, idx)
    np.testing.assert_array_equal(ref[0], X1); assert ref[2][0] == nk1
    bad = [(dict(pairs=[(0, 2)]), "outside \\[0, 2\\)"),
           (dict(pairs=[(-1, 1)]), "outside \\[0, 2\\)"),
           (dict(img_off=[0, len(a) + 10, len(a)]), "img_off is not monotone"),
           (dict(img_off=[1, len(a), len(a) + len(b)]), "img_off\\[0\\] must be 0"),
           (dict(pairs=[(0, 1), (0, 1)], moff=[0, 60, 30]), "match_off is not monotone"),
           (dict(moff=[5, 60]), "match_off\\[0\\] must be 0"),
           (dict(mq=np.r_[idx[:59], len(a)]), "indexes outside its images"),
           (dict(mt=np.r_[-1, idx[1:]]), "indexes outside its images")]
    for change, msg in bad:
        args = {**good, **change}
        poses = np.repeat(pose, len(args["pairs"]), 0)
        with pytest.raises(capi.SfmB200Error, match=msg):
            _raw(ctx, K, poses, [a, b], **args)
        again = _raw(ctx, K, pose, [a, b], **good)
        for x, y in zip(again, ref):
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
