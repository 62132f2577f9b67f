"""cv::findHomography(RANSAC) restated (tests/homography_oracle.py) and pinned to cv2 without a GPU: the RANSAC phase (the refit of
cv2 on the restated inlier set returns cv2's RANSAC H bit for bit), the refinement, the returned counts and masks on the crazyhorse
pairs and on synthetic scenes; then the g++-compiled csrc/homography_math.cuh against the restatement."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from cfg1_util import Cfg1
import homography_oracle as ho
from homography_util import crazyhorse_pairs, synthetic_scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def pairs():
    return crazyhorse_pairs(Cfg1())


@pytest.fixture(scope="module")
def oracle_runs(pairs):
    return [ho.find_homography(a, b) for a, b in pairs]


@pytest.fixture(scope="module")
def hh():
    so = os.path.join(ROOT, "tests", "_build", "libhost_homography.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_homography.cpp"), "-o", so],
                   check=True)
    return C.CDLL(so)


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_ransac_phase_reproduces_cv2(pairs, oracle_runs):
    # cv2 refits and refines on its RANSAC inliers; given the restated inlier set, method 0 does exactly that, so an identical H
    # means the sample sequence, the subset checks, the 4-point kernel and the selection were all reproduced
    for (a, b), o in zip(pairs, oracle_runs):
        H, m = cv2.findHomography(a, b, cv2.RANSAC, 10.0)
        sel = o["ransac_mask"].astype(bool)
        H0, m0 = cv2.findHomography(a[sel], b[sel], 0)
        assert np.array_equal(H0, H)
        assert o["ransac_inliers"] <= o["n_inliers"] and o["iterations"] == len(o["visited"]) > 0


def test_refinement_matches_cv2(pairs, oracle_runs):
    for (a, b), o in zip(pairs, oracle_runs):
        sel = o["ransac_mask"].astype(bool)
        H0, _ = cv2.findHomography(a[sel], b[sel], 0)
        assert np.abs(o["H"] - H0).max() <= 1e-7 * np.abs(H0).max()


def test_counts_and_masks_equal_cv2_on_crazyhorse(pairs, oracle_runs):
    for (a, b), o in zip(pairs, oracle_runs):
        H, m = cv2.findHomography(a, b, cv2.RANSAC, 10.0)
        assert np.array_equal(o["mask"], m.ravel()) and o["n_inliers"] == int(m.sum())


def test_counts_and_masks_equal_cv2_on_synthetic_scenes():
    scenes = synthetic_scenes()
    assert len(scenes) >= 20
    for name, a, b in scenes:
        H, m = cv2.findHomography(a, b, cv2.RANSAC, 10.0)
        o = ho.find_homography(a, b)
        assert (H is None) == (o["H"] is None), name
        if H is not None:
            assert np.array_equal(o["mask"], m.ravel()), name
    assert ho.find_homography(scenes[0][1][:3], scenes[0][2][:3])["n_inliers"] == 0


def test_generator_is_cv_rng():
    r = ho.CvRng()
    # cv::RNG((uint64)-1): state = 0xffffffff * 4164903690 + 0xffffffff
    assert r.next() == (0xFFFFFFFF * 4164903690 + 0xFFFFFFFF) & 0xFFFFFFFF


def test_device_math_draws_the_oracle_quads(hh, pairs):
    cases = [pairs[0], pairs[5], pairs[12]] + [(a, b) for name, a, b in synthetic_scenes() if name in ("planar_n5_out0", "planar_n300_out70", "repeated")]
    for a, b in cases:
        a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b, np.float32)
        idx = np.zeros((2000, 4), np.int32)
        got = hh.host_draw_subsets(_f(a), _f(b), len(a), 2000, idx.ctypes.data_as(C.POINTER(C.c_int)))
        rng = ho.CvRng()
        ref = [ho.get_subset(a, b, rng) for _ in range(2000)]
        assert got == 2000 and np.array_equal(idx, np.array(ref))
        line = np.ascontiguousarray(np.c_[np.arange(10), 2 * np.arange(10)], np.float32)
        assert hh.host_draw_subsets(_f(line), _f(line), 10, 1, idx.ctypes.data_as(C.POINTER(C.c_int))) == 0


def test_device_math_kernel_and_refinement(hh, pairs, oracle_runs):
    # The 4-point solutions: the eigenvector of the smallest eigenvalue of L^T L carries the squared condition number of the
    # sample, so two correct solvers (cv2's Jacobi, numpy's eigh, ours) differ by up to ~1e-8 of max|H| on these samples;
    # cv2.getPerspectiveTransform on the same quads differs from cv2's DLT by up to 1.7e-3.
    worst = 0.0
    for a, b in pairs[:6]:
        rng = ho.CvRng()
        for _ in range(100):
            q = ho.get_subset(a, b, rng)
            A = np.ascontiguousarray(a[q]); B = np.ascontiguousarray(b[q]); H = np.zeros(9)
            assert hh.host_kernel(_f(A), _f(B), 4, _d(H)) == 1
            Hc, _ = cv2.findHomography(A, B, 0)
            worst = max(worst, np.abs(H.reshape(3, 3) - Hc).max() / np.abs(Hc).max())
    assert worst < 1e-7, worst
    same = np.zeros((4, 2), np.float32); H = np.zeros(9)
    assert hh.host_kernel(_f(same), _f(same), 4, _d(H)) == 0
    for (a, b), o in zip(pairs, oracle_runs):
        sel = o["ransac_mask"].astype(bool)
        A = np.ascontiguousarray(a[sel]); B = np.ascontiguousarray(b[sel]); H = np.zeros(9); Hr = np.zeros(9)
        assert hh.host_kernel(_f(A), _f(B), len(A), _d(H)) == 1
        hh.host_refine(_f(A), _f(B), len(A), _d(H), 10, _d(Hr))
        H0, _ = cv2.findHomography(A, B, 0)
        assert np.abs(Hr.reshape(3, 3) - H0).max() <= 1e-6 * np.abs(H0).max()
        assert np.array_equal(ho.err_homography(Hr, a, b) <= np.float32(100), o["mask"].astype(bool))
