"""The five-point solver, sample drawing and E decomposition of csrc/essential_math.cuh (__host__ __device__) compiled with g++ and
checked against cv2 without a GPU; the generated coefficient header against its generator; the oracle's restatement of OpenCV's
sequential RANSAC loop on hand-computed cases."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from cfg1_util import Cfg1
from essential_util import canon, compare_with_cv2, five_point_samples
import essential_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def he():
    so = os.path.join(ROOT, "tests", "_build", "libhost_essential.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_essential.cpp"), "-o", so],
                   check=True)
    return C.CDLL(so)


def _solve(he, x1, x2):
    x1 = np.ascontiguousarray(x1, np.float64); x2 = np.ascontiguousarray(x2, np.float64)
    ns = len(x1); E = np.zeros((ns, 10, 9)); n = np.zeros(ns, np.int32)
    he.host_five_point(_d(x1), _d(x2), ns, _d(E), n.ctypes.data_as(C.POINTER(C.c_int)))
    return E, n


def test_five_point_matches_cv2(he):
    x1, x2, A, B = five_point_samples(Cfg1())
    E, n = _solve(he, x1, x2)
    same, unmatched, epi, con = compare_with_cv2(cv2, x1, x2, A, B, E, n)
    assert same >= 0.99, same
    assert unmatched == 0
    assert epi < 1e-9 and con < 1e-9, (epi, con)
    assert np.all(np.isfinite(E))


def test_five_point_solution_counts_vary_on_pair0(he):
    cfg = Cfg1(); rs = np.random.RandomState(1)
    i, j = cfg.pairs[0]; q, t, _ = cfg.matches[0]
    a = cfg.features[i].points[q].astype(np.float64); b = cfg.features[j].points[t].astype(np.float64)
    idx = np.array([rs.choice(len(a), 5, replace=False) for _ in range(300)])
    E, n = _solve(he, (a[idx] - [512, 384]) / 2500.0, (b[idx] - [512, 384]) / 2500.0)
    counts = np.bincount(n, minlength=11)
    assert (counts > 20).sum() >= 3, counts             # cv2 on its own 300 samples: 2 / 4 / 6 solutions 33 / 135 / 132 times


def test_five_point_degenerate_samples_give_no_solution(he):
    x = np.tile(np.array([[0.1, -0.05]]), (5, 1))[None]
    E, n = _solve(he, x, x)
    assert n[0] == 0
    rs = np.random.RandomState(0)
    x1 = rs.normal(0, 0.2, (1, 5, 2)); x2 = x1.copy(); x2[0, 3] = x2[0, 1]; x1[0, 3] = x1[0, 1]    # a repeated correspondence
    E, n = _solve(he, x1, x2)
    assert n[0] == 0 and np.all(np.isfinite(E))


def test_decomposition_matches_cv2(he):
    rs = np.random.RandomState(5)
    for _ in range(50):
        from essential_util import rot
        Rt = rot(rs.normal(0, 0.5, 3)); t = rs.normal(0, 1, 3); t /= np.linalg.norm(t)
        E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ Rt
        E = np.ascontiguousarray(E / np.linalg.norm(E) * rs.choice([-1, 1]))
        R1 = np.zeros(9); R2 = np.zeros(9); tt = np.zeros(3)
        assert he.host_decompose(_d(E), _d(R1), _d(R2), _d(tt)) == 1
        c1, c2, ct = cv2.decomposeEssentialMat(E)
        ours = sorted([R1.reshape(3, 3), R2.reshape(3, 3)], key=lambda r: r[0, 0]); theirs = sorted([c1, c2], key=lambda r: r[0, 0])
        np.testing.assert_allclose(ours[0], theirs[0], atol=1e-12); np.testing.assert_allclose(ours[1], theirs[1], atol=1e-12)
        assert min(np.abs(tt - ct.ravel()).max(), np.abs(tt + ct.ravel()).max()) < 1e-12


def test_samples_are_distinct_in_range_and_deterministic(he):
    idx = np.zeros(5, np.int32); p = idx.ctypes.data_as(C.POINTER(C.c_int))
    seen = []
    for n in (5, 6, 37, 1159):
        for s in range(200):
            he.host_sample(C.c_ulonglong(7), s, n, p)
            assert len(set(idx.tolist())) == 5 and idx.min() >= 0 and idx.max() < n
            seen.append(idx.copy())
    he.host_sample(C.c_ulonglong(7), 199, 1159, p)
    np.testing.assert_array_equal(idx, seen[-1])
    he.host_sample(C.c_ulonglong(8), 199, 1159, p)
    assert not np.array_equal(idx, seen[-1])


def test_generated_header_is_reproducible(tmp_path):
    path = os.path.join(ROOT, "sfm-toy-library_b200", "csrc", "five_point.cuh")
    committed = open(path, "rb").read()
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    src = open(os.path.join(ROOT, "tools", "gen_five_point.py")).read().replace(
        'OUT = os.path.join(ROOT, "sfm-toy-library_b200", "csrc", "five_point.cuh")', "OUT = %r" % str(tmp_path / "five_point.cuh"))
    script = tmp_path / "gen.py"
    script.write_text(src)
    subprocess.run([sys.executable, str(script)], check=True, env=env, capture_output=True)
    assert (tmp_path / "five_point.cuh").read_bytes() == committed


def test_update_num_iters_hand_computed():
    # log(0.001) / log(1 - 0.5^5) = 217.57
    assert eo.ransac_update_num_iters(0.999, 0.5, 5, 1000) == 218
    # log(0.001) / log(1 - 0.8^5) = 17.40
    assert eo.ransac_update_num_iters(0.999, 0.2, 5, 1000) == 17
    assert eo.ransac_update_num_iters(0.999, 0.0, 5, 1000) == 0          # no outliers: 1 - (1 - 0)^5 = 0 < DBL_MIN
    assert eo.ransac_update_num_iters(0.999, 0.9, 5, 1000) == 1000       # would need 690 772 samples: capped
    assert eo.ransac_update_num_iters(0.999, 0.5, 5, 100) == 100         # the cap is the current budget
    assert eo.ransac_update_num_iters(0.999, 1.5, 5, 1000) == 1000       # ep clamped to 1: log(1 - 0) = 0 >= 0
    assert eo.ransac_update_num_iters(1.0, 0.5, 5, 1000) == 1000         # p = 1: num = log(DBL_MIN), over the cap


def test_sequential_select_hand_computed():
    # sample 0: counts 3, 4 (not > 4); sample 1: 10 (best, budget -> ...); sample 2: 10 (tie: the earlier stays), 12 (best)
    nsol = [2, 1, 2, 0, 1]; counts = [3, 4, 10, 10, 12, 5]
    best, good, it = eo.sequential_select(nsol, counts, 20)
    assert (best, good, it) == (4, 12, 5)
    # everything an inlier: the budget drops to 0 after the first improvement; the rest of that sample is still visited
    best, good, it = eo.sequential_select([3, 4], [20, 19, 20, 20, 20, 20, 20], 20)
    assert (best, good, it) == (0, 20, 1)
    assert eo.sequential_select([2, 2], [4, 1, 0, 4], 20) == (-1, 0, 2)
