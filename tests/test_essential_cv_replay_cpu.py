"""The Python replay of cv::findEssentialMat(RANSAC) (tests/essential_cv_replay.py: cv::RNG restarted at (uint64)-1, getSubset's
redraws, cv2's five-point solutions per sample, the pinned scoring and the sequential loop) against cv2.findEssentialMat itself,
without a GPU: on every crazyhorse pair and on synthetic scenes the replay's winner is cv2's E, its mask is cv2's mask, and its
iteration count is what the pinned selection loop returns on the replay's counts.  This pins the sample sequence the device's
OpenCV sampler reproduces."""
import numpy as np
import pytest

from cfg1_util import Cfg1
import essential_oracle as eo
from essential_cv_replay import CvRng, cv_samples, replay, synthetic_cases
from essential_util import CX, CY, F, canon, synthetic_scene

cv2 = pytest.importorskip("cv2")


def _check(a, b, label):
    r = replay(cv2, a, b, F, (CX, CY))
    Ec, mc = cv2.findEssentialMat(a, b, F, (CX, CY), cv2.RANSAC, 0.999, 1.0)
    assert r["best"] >= 0 and Ec is not None, label
    # m == 5: cv2 stacks every solution of the one sample; the replay's winner is one of them
    d = min(np.abs(canon(r["E"]) - canon(Ec[3 * k:3 * k + 3])).max() for k in range(Ec.shape[0] // 3))
    assert d < 1e-9, (label, d)
    if len(a) > 5:
        np.testing.assert_array_equal(r["mask"], mc.ravel(), err_msg=label)
        assert r["n_inliers"] == int(mc.sum()), label
    assert eo.sequential_select(r["nsol"], r["counts"], len(a)) == (r["best"], r["n_inliers"], r["iterations"]), label
    np.testing.assert_array_equal(r["samples"], cv_samples(len(a), r["iterations"]), err_msg=label)
    return r


def test_cv_rng_first_draws():
    # state 2^64-1: (2^32-1) * 4164903690 + (2^32-1) = 4164903690 * 2^32 - 4164903690 + 2^32 - 1
    rng = CvRng()
    s1 = (0xFFFFFFFF * 4164903690 + 0xFFFFFFFF) & ((1 << 64) - 1)
    assert rng.next() == s1 & 0xFFFFFFFF
    assert rng.state == s1
    s2 = (s1 & 0xFFFFFFFF) * 4164903690 + (s1 >> 32)
    assert rng.next() == s2 & 0xFFFFFFFF


def test_samples_are_distinct_and_in_range():
    for n in (5, 6, 7, 9, 37, 1159):
        s = cv_samples(n, 300)
        assert s.min() >= 0 and s.max() < n
        assert all(len(set(r.tolist())) == 5 for r in s)
    np.testing.assert_array_equal(cv_samples(5, 1), [[0, 1, 2, 3, 4]])
    np.testing.assert_array_equal(cv_samples(300, 40), cv_samples(300, 100)[:40])     # a prefix of one stream


def test_replay_is_cv2_on_every_crazyhorse_pair():
    cfg = Cfg1()
    visited = []
    for p, (i, j) in enumerate(cfg.pairs):
        q, t, _ = cfg.matches[p]
        r = _check(cfg.features[i].points[q], cfg.features[j].points[t], f"pair {p}")
        visited.append(r["iterations"])
    assert 20 <= min(visited) and max(visited) <= 400, visited


def test_replay_is_cv2_on_synthetic_scenes():
    its = []
    for seed, n, out in synthetic_cases():
        a, b, *_ = synthetic_scene(seed, n, noise_px=0.5, outliers=out)
        its.append(_check(a, b, f"scene {seed} n {n} outliers {out}")["iterations"])
    assert min(its) < 20 and max(its) == 1000, its                # early stops and budget-bound runs both covered


@pytest.mark.parametrize("n", [5, 6, 7, 9])
def test_replay_is_cv2_on_tiny_sets(n):
    a, b, *_ = synthetic_scene(40 + n, n, noise_px=0.5)
    r = _check(a, b, f"n {n}")
    if n == 5:
        assert r["iterations"] == 1 and r["samples"].tolist() == [[0, 1, 2, 3, 4]]
