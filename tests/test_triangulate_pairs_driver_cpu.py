"""The driver mirror with a batched triangulation stage (runsfm.SfM(triangulateManyPairs=...)), on the CPU.  The crazyhorse replay
runs with the CPU stages of tools/bench_cfg1.py's cpu arm (oracle.cv2_stages) and cv2's findEssentialMat / recoverPose, which seed
their own RNG on every call.  One run triangulates pair by pair; the other hands the driver a batched function that calls
cv2_stages.triangulateViews for each pair of its batch.  Both runs must agree in every trace entry, in the match lists every
mergeNewPointCloud sees and in the final state: the batch is computed before the walk, and each pair's pruned list may still only
be stored at that pair's own turn."""
import numpy as np
import pytest

from cfg1_util import Cfg1

cv2 = pytest.importorskip("cv2")


def _replay(batched_triangulation, batched_essential=False):
    from oracle import cv2_stages
    from sfm_toy_library_b200 import runsfm
    from sfm_toy_library_b200.stages import ImagePair
    cfg1 = Cfg1()
    per_pair = runsfm.findCameraMatricesFromMatch_cv2
    kw = dict(matchFeatures=cv2_stages.matchFeatures, triangulateViews=cv2_stages.triangulateViews,
              adjustBundle=lambda *a: cv2_stages.adjustBundle(*a, num_threads=1), findCameraMatricesFromMatch=per_pair)
    if batched_essential:
        kw["findCameraMatricesManyPairs"] = lambda intr, f, pairs, matches: [per_pair(intr, m, f[i], f[j]) for (i, j), m in zip(pairs, matches)]
    batches = []
    if batched_triangulation:
        def many(intrinsics, features, pairs, matches, poses):
            batches.append(list(pairs))
            clouds = []
            for (i, j), m, (Pl, Pr) in zip(pairs, matches, poses):
                cloud = []
                assert cv2_stages.triangulateViews(intrinsics, ImagePair(i, j), m, features[i], features[j], Pl, Pr, cloud)
                clouds.append(cloud)
            return clouds
        kw["triangulateManyPairs"] = many
    trace = []
    sfm = runsfm.SfM(cfg1.features, cfg1.size, trace=trace, **kw)
    merges = []
    merge = sfm.mergeNewPointCloud

    def recording_merge(cloud):
        merges.append([len(sfm.mFeatureMatchMatrix[l][r]) for l in range(sfm.n) for r in range(l + 1, sfm.n)])
        return merge(cloud)
    sfm.mergeNewPointCloud = recording_merge
    sfm.runSfM()
    return sfm, trace, merges, batches


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


@pytest.fixture(scope="module")
def per_pair_run(oracle):
    return _replay(batched_triangulation=False)


@pytest.mark.parametrize("batched_essential", [False, True])
def test_batched_triangulation_stage_replays_the_per_pair_driver(per_pair_run, batched_essential):
    seq, seq_trace, seq_merges, _ = per_pair_run
    bat, bat_trace, bat_merges, batches = _replay(batched_triangulation=True, batched_essential=batched_essential)
    # one batch per view added after a successful PnP; the baseline keeps its single triangulateViews call
    n_added = sum(1 for e in seq_trace if e["stage"] == "pnp" and e["ok"])
    assert n_added > 0 and len(batches) == n_added
    assert bat.calls["triangulate"] == 1 + n_added
    assert seq.calls["triangulate"] == 1 + sum(len(b) for b in batches)
    _assert_same(seq_trace, bat_trace, "trace")
    assert len(seq_merges) > 0
    _assert_same(seq_merges, bat_merges, "match list lengths at each mergeNewPointCloud")
    np.testing.assert_array_equal(np.array([p.p for p in seq.mReconstructionCloud]), np.array([p.p for p in bat.mReconstructionCloud]))
    assert [p.originatingViews for p in seq.mReconstructionCloud] == [p.originatingViews for p in bat.mReconstructionCloud]
    np.testing.assert_array_equal(np.array(seq.mCameraPoses), np.array(bat.mCameraPoses))
    np.testing.assert_array_equal(seq.mIntrinsics.K, bat.mIntrinsics.K)
    for l in range(seq.n):
        for r in range(seq.n):
            np.testing.assert_array_equal(seq.mFeatureMatchMatrix[l][r], bat.mFeatureMatchMatrix[l][r], err_msg=f"matches {l},{r}")
