"""TEST INFRASTRUCTURE ONLY: a replay of cv::findEssentialMat(RANSAC) in Python, sample by sample, built from pieces that are
each pinned to cv2 on their own.  OpenCV 4.x (calib3d ptsetreg.cpp, five-point.cpp) runs RANSACPointSetRegistrator::run with:
  * a fresh cv::RNG((uint64)-1) on every call: multiply-with-carry, state = (uint32)state * 4164903690 + (state >> 32), each draw
    the low 32 bits, rng.uniform(0, n) = draw % n;
  * getSubset: five indices drawn one after another, an index that repeats an earlier one of the same sample redrawn;
    EMEstimatorCallback has no subset check, so the sequence depends on the number of matches only;
  * every sample solved by the five-point kernel: cv2.findEssentialMat on exactly those 5 points returns all its solutions in
    OpenCV's order (its model_points == count branch);
  * every solution scored with EMEstimatorCallback's error and inlier rule (oracle/ransac_oracle.score(1, ..., 1 / focal));
  * the sequential loop of essential_oracle.sequential_select, one sample at a time.
With m == 5 there is no drawing: the kernel runs once on the five points in their order."""
import numpy as np

import essential_oracle as eo
from oracle import ransac_oracle as ro

_M64 = (1 << 64) - 1
CV_RNG_COEFF = 4164903690


class CvRng:
    """cv::RNG seeded with (uint64)-1, as RANSACPointSetRegistrator::run seeds it."""

    def __init__(self, state=_M64):
        self.state = state

    def next(self):
        self.state = ((self.state & 0xFFFFFFFF) * CV_RNG_COEFF + (self.state >> 32)) & _M64
        return self.state & 0xFFFFFFFF

    def uniform(self, n):
        return self.next() % n


def cv_samples(n, count, k=5):
    """The first `count` index sets getSubset draws for n matches (no subset check): [count, k] int32.  n == k: the one
    sample of the model_points == count branch, 0 .. k-1."""
    if n == k:
        return np.arange(k, dtype=np.int32).reshape(1, k)[:count]
    rng = CvRng(); out = np.zeros((count, k), np.int32)
    for s in range(count):
        idx = []
        while len(idx) < k:
            v = rng.uniform(n)
            if v not in idx:
                idx.append(v)
        out[s] = idx
    return out


def solve_sample(cv2, a, b, idx, focal, pp):
    """cv2's five-point solutions of one sample, in OpenCV's order: [nsol, 9]"""
    E, _ = cv2.findEssentialMat(np.ascontiguousarray(a[idx], np.float64), np.ascontiguousarray(b[idx], np.float64), focal, pp,
                                cv2.RANSAC, 0.999, 1.0)
    return np.zeros((0, 9)) if E is None else E.reshape(-1, 3, 3).reshape(-1, 9)


def replay(cv2, a, b, focal, pp, max_iters=1000, confidence=0.999, threshold_px=1.0):
    """findEssentialMat(a, b, focal, pp, RANSAC, confidence, threshold_px) replayed.  Returns a dict: samples [it, 5] (the visited
    ones), nsol [it], counts [sum nsol], hyps [sum nsol, 9], best (index into hyps or -1), E [3, 3] (zeros without a model),
    mask [m] uint8, n_inliers, iterations."""
    a = np.asarray(a, np.float32).reshape(-1, 2); b = np.asarray(b, np.float32).reshape(-1, 2)
    m = len(a); aux = (focal, pp[0], pp[1])
    samples, nsol, counts, hyps = [], [], [], []
    niters = max(max_iters, 1); best = -1; max_good = 0; it = 0
    rng = CvRng()
    while it < niters and m >= 5:
        if m == 5:
            idx = list(range(5))
        else:
            idx = []
            while len(idx) < 5:
                v = rng.uniform(m)
                if v not in idx:
                    idx.append(v)
        H = solve_sample(cv2, a, b, np.array(idx), focal, pp)
        c = ro.score(1, a, b, H, aux, threshold_px / focal)[0] if len(H) else np.zeros(0, np.int32)
        for k in range(len(H)):
            if c[k] > max(max_good, 4):
                best = len(hyps) + k; max_good = int(c[k])
                niters = eo.ransac_update_num_iters(confidence, (m - max_good) / m, 5, niters)
        samples.append(idx); nsol.append(len(H)); counts.extend(int(x) for x in c); hyps.extend(H)
        it += 1
        if m == 5:
            break
    hyps = np.array(hyps, np.float64).reshape(-1, 9)
    E = hyps[best].reshape(3, 3) if best >= 0 else np.zeros((3, 3))
    mask = ro.score(1, a, b, E.reshape(1, 9), aux, threshold_px / focal)[2] if best >= 0 else np.zeros(m, np.uint8)
    return dict(samples=np.array(samples, np.int32).reshape(-1, 5), nsol=np.array(nsol, np.int32), counts=np.array(counts, np.int32),
                hyps=hyps, best=best, E=E, mask=mask, n_inliers=max_good if best >= 0 else 0, iterations=it)



def synthetic_cases():
    """(seed, n, outlier ratio) of the synthetic scenes (essential_util.synthetic_scene at 0.5 px noise): n = 60 .. 1200, 0 - 70 %
    outliers"""
    return [(k, n, o) for k, (n, o) in enumerate((n, o) for n in (60, 100, 200, 400, 800, 1200) for o in (0.0, 0.3, 0.5, 0.7))]
