"""SURVEY.md 8(f-1) on the device: find2D3DMatches and mergeNewPointCloud (SfM.cpp:471-600) through sfmb200_find_2d3d_matches /
sfmb200_merge_point_cloud.

  (i)   the C++ DeviceGlue (host/sfm_glue_device.cpp) against host/sfm_glue.cpp on every scene test_glue uses (6 matcher-like,
        6 adversarial, the empty scene, the bench scene), on hand-built scenes for each ordering rule of the merge, on lists
        replaced with setPair, and the C ABI's refusals (the context stays usable after each);
  (ii)  stages.find2D3DMatches / stages.mergeNewPointCloud against runsfm.SfM's own Python loops on random scenes;
  (iii) the crazyhorse replay with the device glue injected gives the trace of the default replay.
"""
import copy
import os
import subprocess

import numpy as np
import pytest

from sfm_toy_library_b200 import capi, runsfm, stages
from sfm_toy_library_b200.stages import DMATCH, Features, Point3DInMap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _exe():
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_glue_device")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    return exe


@pytest.mark.parametrize("seed", [1, 5])
def test_cpp_device_glue_equals_host_glue(seed):
    r = subprocess.run([_exe(), str(seed)], capture_output=True, text=True, timeout=600)
    print(r.stdout[-4000:], r.stderr[-2000:])
    assert r.returncode == 0 and "all device-glue checks passed" in r.stdout
    # 12 random scenes, the empty and the bench scene, 5 hand-built scenes, 2 setPair checks
    assert sum(1 for l in r.stdout.splitlines() if l.startswith("ok ") and not l.startswith("ok refusal")) == 21
    assert sum(1 for l in r.stdout.splitlines() if l.startswith("ok refusal")) == 26


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    stages._GlueIndex.state = None
    c.close()


def _scene(seed, V, F, n_recon, n_new, matcher_like):
    rs = np.random.RandomState(seed)
    feats = [Features(points=rs.uniform(0, 1000, (F, 2)).astype(np.float32)) for _ in range(V)]
    M = [[np.zeros(0, DMATCH) for _ in range(V)] for _ in range(V)]
    for i in range(V):
        for j in range(i + 1, V):
            if matcher_like:
                q = np.nonzero(rs.rand(F) < 0.35)[0]
                t = rs.randint(0, F, len(q))
            else:
                q = rs.randint(0, F // 4, F // 2); t = rs.randint(0, F // 4, F // 2)
            m = np.zeros(len(q), DMATCH)
            m["queryIdx"] = q; m["trainIdx"] = t; m["distance"] = rs.randint(0, 50, len(q)).astype(np.float32)
            M[i][j] = m
    hi = F if matcher_like else F // 4

    def views():
        vs = rs.choice(V, rs.randint(2, 5), replace=False)
        return {int(v): int(rs.randint(0, hi)) for v in vs}
    recon = [Point3DInMap(rs.uniform([-1, -1, 4], [1, 1, 6]).astype(np.float32), views()) for _ in range(n_recon)]
    fresh = []
    for _ in range(n_new):
        mode = rs.randint(0, 4)
        if mode == 0 or not recon:
            fresh.append(Point3DInMap(rs.uniform([-1, -1, 4], [1, 1, 6]).astype(np.float32), views()))
            continue
        e = recon[rs.randint(len(recon))]
        p = (e.p + rs.uniform(-1, 1, 3) * (0.004 if mode == 1 else 0.012)).astype(np.float32)
        v = views()
        if mode != 3:                                       # a likely confirming match with one of e's views
            ev = int(rs.choice(sorted(e.originatingViews)))
            nv = int(rs.randint(V))
            nv = (nv + 1) % V if nv == ev else nv
            l, r = min(nv, ev), max(nv, ev)
            if len(M[l][r]):
                d = M[l][r][rs.randint(len(M[l][r]))]
                v = {nv: int(d["queryIdx"] if nv == l else d["trainIdx"])}
                e.originatingViews[ev] = int(d["queryIdx"] if ev == l else d["trainIdx"])
                v[int(rs.randint(V))] = int(rs.randint(0, hi))
        fresh.append(Point3DInMap(p, v))
    done = {v for v in range(V) if rs.rand() < 0.5}
    return feats, M, recon, fresh, done


def _sfm(feats, M, recon, done):
    sfm = runsfm.SfM(feats, (1024, 768))
    sfm.mFeatureMatchMatrix = M
    sfm.mReconstructionCloud = recon
    sfm.mDoneViews = set(done)
    return sfm


@pytest.mark.parametrize("seed,matcher_like", [(s, m) for s in range(4) for m in (True, False)])
def test_stages_equal_the_python_glue(ctx, seed, matcher_like):
    feats, M, recon, fresh, done = _scene(100 + seed, 5 + seed, 120 if matcher_like else 60, 500, 400, matcher_like)
    sfm = _sfm(feats, M, copy.deepcopy(recon), done)
    want = sfm.find2D3DMatches()
    got = stages.find2D3DMatches(len(feats), done, M, feats, recon, ctx=ctx)
    assert sorted(want) == sorted(got)
    for v in want:
        np.testing.assert_array_equal(want[v][0], got[v][0]); np.testing.assert_array_equal(want[v][1], got[v][1])
    a_new, b_new = copy.deepcopy(fresh), copy.deepcopy(fresh)
    counts_want = sfm.mergeNewPointCloud(a_new)
    b_recon = copy.deepcopy(recon)
    counts_got = stages.mergeNewPointCloud(b_new, b_recon, M, feats, ctx=ctx)
    assert counts_want == counts_got and counts_want[1] > 0
    a_recon = sfm.mReconstructionCloud
    assert len(a_recon) == len(b_recon)
    for p, q in zip(a_recon, b_recon):
        assert np.asarray(p.p, np.float32).tobytes() == np.asarray(q.p, np.float32).tobytes() and p.originatingViews == q.originatingViews
    # a replaced list (SfM.cpp:431) reaches the device index before the next call
    M[0][2] = M[0][2][::2].copy()
    sfm.mReconstructionCloud = copy.deepcopy(recon)
    want = sfm.find2D3DMatches()
    got = stages.find2D3DMatches(len(feats), done, M, feats, recon, ctx=ctx)
    for v in want:
        np.testing.assert_array_equal(want[v][0], got[v][0]); np.testing.assert_array_equal(want[v][1], got[v][1])


def _same_value(u, w, where):
    """Bitwise equality of trace values: arrays, lists / tuples of them, scalars.  The bundle-adjustment summary (a dict) holds
    wall-clock times and is skipped; its cost and parameters are in the trace as arrays."""
    if isinstance(u, np.ndarray) or isinstance(w, np.ndarray):
        np.testing.assert_array_equal(u, w, err_msg=where)
    elif isinstance(u, (list, tuple)):
        assert isinstance(w, (list, tuple)) and len(u) == len(w), where
        for i, (a, b) in enumerate(zip(u, w)):
            _same_value(a, b, f"{where}[{i}]")
    elif not isinstance(u, dict):
        assert u == w, where


def _same_trace(a, b):
    assert [e["stage"] for e in a] == [e["stage"] for e in b]
    for n, (x, y) in enumerate(zip(a, b)):
        assert sorted(x) == sorted(y), x["stage"]
        for k in x:
            _same_value(x[k], y[k], f'trace entry {n} ({x["stage"]}) {k}')


def test_crazyhorse_replay_with_device_glue(ctx):
    from cfg1_util import Cfg1
    cfg1 = Cfg1()
    common = dict(matchAllPairs=lambda feats, pairs: stages.matchAllPairs(feats, pairs, ctx=ctx),
                  triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx),
                  adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx))
    runs = []
    for hooks in ({}, dict(find2D3DMatches=lambda *a: stages.find2D3DMatches(*a, ctx=ctx),
                           mergeNewPointCloud=lambda *a: stages.mergeNewPointCloud(*a, ctx=ctx))):
        trace = []
        sfm = runsfm.SfM(cfg1.features, cfg1.size, trace=trace, **common, **hooks)
        sfm.runSfM()
        runs.append((trace, sfm))
    (ta, a), (tb, b) = runs
    assert b.calls["glue"] == a.calls["glue"] > 0
    _same_trace(ta, tb)
    assert len(a.mReconstructionCloud) == len(b.mReconstructionCloud)
    for p, q in zip(a.mReconstructionCloud, b.mReconstructionCloud):
        assert p.originatingViews == q.originatingViews
        np.testing.assert_array_equal(p.p, q.p)
