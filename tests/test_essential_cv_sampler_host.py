"""The OpenCV sampler of csrc/essential_math.cuh (em_cv_samples over csrc/cv_rng.cuh, __host__ __device__) compiled with g++ and
checked without a GPU: its index sequences are the Python replay's (tests/essential_cv_replay.py, pinned to cv2), including tiny
n where redraws are frequent; then the host-compiled sampler, the five-point solver, the scoring restatement and the selection
restatement run end to end against cv2.findEssentialMat on the crazyhorse pairs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from cfg1_util import Cfg1
import essential_oracle as eo
from essential_cv_replay import CvRng, cv_samples, replay
from essential_util import CX, CY, F, canon
from oracle import ransac_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def hc():
    so = os.path.join(ROOT, "tests", "_build", "libhost_essential_cv.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_essential_cv.cpp"), "-o", so],
                   check=True)
    return C.CDLL(so)


def _i(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _samples(hc, m, S):
    out = np.zeros((S, 5), np.int32)
    hc.host_cv_samples(m, S, _i(out))
    return out


def test_raw_stream_is_cv_rng(hc):
    for n in (2, 5, 7, 1000, 2 ** 31 - 1):
        out = np.zeros(500, np.int32)
        hc.host_cv_uniform(n, 500, _i(out))
        rng = CvRng()
        np.testing.assert_array_equal(out, [rng.uniform(n) for _ in range(500)], err_msg=f"n {n}")


@pytest.mark.parametrize("m", [5, 6, 7, 8, 11, 60, 307, 1159, 100000])
def test_samples_are_the_replays(hc, m):
    S = 1 if m == 5 else 1000                    # m == 5: one sample, the five points in order
    np.testing.assert_array_equal(_samples(hc, m, S), cv_samples(m, S))


def test_sample_prefix_does_not_depend_on_the_count(hc):
    np.testing.assert_array_equal(_samples(hc, 6, 3), _samples(hc, 6, 1000)[:3])


def test_end_to_end_against_cv2_on_crazyhorse(hc):
    """sampler -> five_point_solve (ascending roots) -> scoring restatement -> selection restatement, against cv2 and against the
    replay (cv2's own solutions per sample).  Visited samples whose sorted per-solution counts differ from cv2's are printed."""
    cfg = Cfg1()
    differ = []
    for p, (i, j) in enumerate(cfg.pairs):
        q, t, _ = cfg.matches[p]
        a = cfg.features[i].points[q]; b = cfg.features[j].points[t]
        smp = _samples(hc, len(a), 1000)
        x1 = np.ascontiguousarray((a[smp].astype(np.float64) - [CX, CY]) / F); x2 = np.ascontiguousarray((b[smp].astype(np.float64) - [CX, CY]) / F)
        E = np.zeros((1000, 10, 9)); ns = np.zeros(1000, np.int32)
        hc.host_five_point(x1.ctypes.data_as(C.POINTER(C.c_double)), x2.ctypes.data_as(C.POINTER(C.c_double)), 1000,
                           E.ctypes.data_as(C.POINTER(C.c_double)), _i(ns))
        hyps = np.concatenate([E[s, :ns[s]] for s in range(1000)])
        counts = ro.score(1, a, b, hyps, (F, CX, CY), 1.0 / F)[0]
        best, good, it = eo.sequential_select(ns, counts, len(a))
        r = replay(cv2, a, b, F, (CX, CY))
        np.testing.assert_array_equal(smp[:it], r["samples"], err_msg=f"pair {p}")
        off = np.r_[0, np.cumsum(ns)]; roff = np.r_[0, np.cumsum(r["nsol"])]
        for s in range(r["iterations"]):
            ours = sorted(counts[off[s]:off[s + 1]]); theirs = sorted(r["counts"][roff[s]:roff[s + 1]])
            if ours != theirs:
                differ.append((p, s, ours, theirs))
        Ec, mc = cv2.findEssentialMat(a, b, F, (CX, CY), cv2.RANSAC, 0.999, 1.0)
        assert it == r["iterations"] and good == int(mc.sum()), (p, it, r["iterations"], good, int(mc.sum()))
        assert np.abs(canon(hyps[best]) - canon(Ec)).max() < 1e-9, p
        np.testing.assert_array_equal(ro.score(1, a, b, hyps[best:best + 1], (F, CX, CY), 1.0 / F)[2], mc.ravel(), err_msg=f"pair {p}")
    print("visited samples whose per-solution counts differ from cv2's:", len(differ), differ[:10])
