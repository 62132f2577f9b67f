"""The null-vector code of csrc/dlt_math.cuh, compiled with g++, against a 40-digit reference (tests/dlt_util.py), on both of its
paths: the closed form wherever it accepts, the Jacobi SVD everywhere, over scenes that put points on either side of the
closed form's gate and on degenerate two-view geometry.  Then the path split itself on the inputs the GPU tests rely on."""
import numpy as np
import pytest

import dlt_util as du
from cfg1_util import Cfg1
from essential_util import CX, CY, F
from sfm_toy_library_b200 import synth

SWEEP = du.sweep()


@pytest.fixture(scope="module")
def lib():
    return du.host_lib()


def _matrices(sc):
    return du.triangulation_matrices(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"], sc["ptsR"])


@pytest.mark.parametrize("name", [n for n, _ in SWEEP])
def test_both_paths_against_the_exact_reference(lib, name):
    A = _matrices(dict(SWEEP)[name])
    idx = du.subsample(len(A), 100)
    A = A[idx]
    vf, ok, vj = du.host_null_vectors(A)
    ref = du.exact(A)
    rj = du.error_ratio(du.dehomogenise(vj), A, ref)
    assert rj.max() <= 1.0, (name, rj.max(), np.argmax(rj))
    if ok.any():
        rf = du.error_ratio(du.dehomogenise(vf[ok]), A[ok], {k: v[ok] for k, v in ref.items()})
        assert rf.max() <= 1.0, (name, rf.max())
    # the gate never accepts what lies 100x below its threshold, and the double margin sorts points as the exact one does
    assert not ok[ref["g"] <= du.FALLBACK_G].any()
    np.testing.assert_array_equal(du.path(du.gate_margin(A), ok), du.path(ref, ok))


def test_rank_deficient_points_lie_in_the_null_space(lib):
    for name in ("identical", "epipole 0 px"):
        A = _matrices(dict(SWEEP)[name])[:200]
        ref = du.exact(A)
        s = ref["sigma"]
        assert (s[:, 2] - s[:, 3] <= du.RANK_DEFICIENT * s[:, 0]).all(), name
        vf, ok, vj = du.host_null_vectors(A)
        assert du.error_ratio(du.dehomogenise(vj), A, ref).max() <= 1.0
        if ok.any():
            assert du.error_ratio(du.dehomogenise(vf[ok]), A[ok], {k: v[ok] for k, v in ref.items()}).max() <= 1.0


def _suite_triangulation_inputs(golden):
    p = synth.make_triangulation_problem(200_000, seed=3)
    yield "make_triangulation_problem", du.triangulation_matrices(p["K"], p["Pl"], p["Pr"], p["ptsL"], p["ptsR"])
    g = golden("triangulate_cv2.npz")
    for pre in ("fx", "sy", "ch"):
        L, R = g[f"{pre}_ptsL"], g[f"{pre}_ptsR"]
        if f"{pre}_mq" in g.files:
            L, R = L[g[f"{pre}_mq"]], R[g[f"{pre}_mt"]]
        yield pre, du.triangulation_matrices(g[f"{pre}_K"], g[f"{pre}_Pl"], g[f"{pre}_Pr"], L, R)
    c = Cfg1()
    for k in range(c.n_tri):
        t = c.tri(k); i, j = (int(x) for x in t["pair"])
        yield f"crazyhorse call {k}", du.triangulation_matrices(t["K"], t["Pl"], t["Pr"], c.features[i].points[t["mq"]],
                                                                c.features[j].points[t["mt"]])


def test_current_suite_inputs_take_the_closed_form(lib, golden):
    cv2 = pytest.importorskip("cv2")
    n = 0
    for name, A in _suite_triangulation_inputs(golden):
        _, ok, _ = du.host_null_vectors(A)
        assert ok.all(), (name, int((~ok).sum()))
        n += len(A)
    assert n > 200_000
    # the cheirality solves of recoverPose on the crazyhorse pairs, all four candidates
    c = Cfg1(); n = 0
    for p in range(len(c.pairs)):
        i, j = c.pairs[p]; q, t, _ = c.matches[p]
        a = c.features[i].points[q].astype(np.float64); b = c.features[j].points[t].astype(np.float64)
        E, _ = cv2.findEssentialMat(a, b, F, (CX, CY), cv2.RANSAC, 0.999, 1.0)
        R1, R2, tt = cv2.decomposeEssentialMat(E[:3])
        for Rc, tc in ((R1, tt), (R2, tt), (R1, -tt), (R2, -tt)):
            _, ok, _ = du.host_null_vectors(du.cheirality_matrices(a, b, F, CX, CY, np.c_[Rc, tc.ravel()]))
            assert ok.all(), (p, int((~ok).sum()))
            n += len(a)
    assert n > 40_000


def test_path_split_on_the_gpu_scenes(lib):
    # fixture x100 and the scene 1000 units from the origin: the fallback for >= 99 % of points, 100x below the gate
    for sc in (du.fixture_scaled(100, 20_000), du.offset_scene(1000.0, 20_000)):
        A = _matrices(sc)
        _, ok, _ = du.host_null_vectors(A)
        assert (du.path(du.gate_margin(A), ok) == "fallback").mean() >= 0.99
    # fixture x10: both paths inside single warps of 32 consecutive points
    A = _matrices(du.fixture_scaled(10, 32 * 200))
    _, ok, _ = du.host_null_vectors(A)
    w = ok.reshape(-1, 32)
    mixed = w.any(1) & ~w.all(1)
    assert mixed.mean() > 0.5, mixed.mean()
    # unit scale: every point on the closed form, 100x above the gate
    A = _matrices(du.fixture_scaled(1, 20_000))
    _, ok, _ = du.host_null_vectors(A)
    assert (du.path(du.gate_margin(A), ok) == "fast").all()
