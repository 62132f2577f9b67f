"""TEST INFRASTRUCTURE ONLY: numpy restatement of cv::findHomography(RANSAC) as OpenCV 4.x computes it (calib3d fundam.cpp,
ptsetreg.cpp, levmarq.cpp), step for step, so that every intermediate of the device implementation (csrc/homography.cu) can
be compared with it:
  * the RANSAC phase: cv::RNG seeded with (uint64)-1 on every call, getSubset (redraw repeated indices, haveCollinearPoints on
    both point sets, the orientation-consistency check of the four triples), the normalised 4-point DLT
    (HomographyEstimatorCallback::runKernel), the sequential selection with RANSACUpdateNumIters;
  * the refinement: the same kernel on the RANSAC inliers, then the Levenberg-Marquardt loop of LMSolverImpl on h00..h21;
  * the final mask: the float transfer error of the refined H against (float)(thr * thr).
Nothing in the product path imports this module."""
import numpy as np

from essential_oracle import ransac_update_num_iters
from oracle.ransac_oracle import err_homography

FLT_EPSILON = float(np.finfo(np.float32).eps)
DBL_EPSILON = float(np.finfo(np.float64).eps)
MASK64 = (1 << 64) - 1


class CvRng:
    """cv::RNG: multiply-with-carry, state = (uint32)state * 4164903690 + (state >> 32)."""

    def __init__(self, state=MASK64):
        self.s = state

    def next(self):
        self.s = ((self.s & 0xFFFFFFFF) * 4164903690 + (self.s >> 32)) & MASK64
        return self.s & 0xFFFFFFFF

    def uniform(self, n):
        return self.next() % n


def _collinear(p):
    """haveCollinearPoints for the last of four points: differences in float, the test in double."""
    i = 3
    for j in range(i):
        dx1 = float(np.float32(p[j, 0] - p[i, 0])); dy1 = float(np.float32(p[j, 1] - p[i, 1]))
        for k in range(j):
            dx2 = float(np.float32(p[k, 0] - p[i, 0])); dy2 = float(np.float32(p[k, 1] - p[i, 1]))
            if abs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (abs(dx1) + abs(dy1) + abs(dx2) + abs(dy2)):
                return True
    return False


def _det3(p, t):
    a = [(float(p[k, 0]), float(p[k, 1]), 1.0) for k in t]
    return (a[0][0] * (a[1][1] * a[2][2] - a[2][1] * a[1][2]) - a[0][1] * (a[1][0] * a[2][2] - a[2][0] * a[1][2])
            + a[0][2] * (a[1][0] * a[2][1] - a[2][0] * a[1][1]))


def check_subset(s, d):
    if _collinear(s) or _collinear(d):
        return False
    neg = sum(1 for t in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (1, 3, 0)) if _det3(s, t) * _det3(d, t) < 0)
    return neg == 0 or neg == 4


def get_subset(a, b, rng, max_attempts=10000):
    """getSubset: four indices, each redrawn while it repeats an earlier one; the whole quad is redrawn when the check fails.
    Returns the quad or None."""
    n = len(a)
    for _ in range(max_attempts):
        idx = []
        for _k in range(4):
            v = rng.uniform(n)
            while v in idx:
                v = rng.uniform(n)
            idx.append(v)
        if check_subset(a[idx], b[idx]):
            return idx
    return None


def ltl(a, b):
    """Normalisation and the 9x9 L^T L of HomographyEstimatorCallback::runKernel.  Returns (LtL, invHnorm, Hnorm2) or None."""
    M = np.asarray(a, np.float32).astype(np.float64); m = np.asarray(b, np.float32).astype(np.float64)
    count = len(M)
    cm = m.sum(0) / count; cM = M.sum(0) / count
    sm = np.abs(m - cm).sum(0); sM = np.abs(M - cM).sum(0)
    if min(abs(sm[0]), abs(sm[1]), abs(sM[0]), abs(sM[1])) < DBL_EPSILON:
        return None
    sm = count / sm; sM = count / sM
    invHnorm = np.array([[1 / sm[0], 0, cm[0]], [0, 1 / sm[1], cm[1]], [0, 0, 1]])
    Hnorm2 = np.array([[sM[0], 0, -cM[0] * sM[0]], [0, sM[1], -cM[1] * sM[1]], [0, 0, 1]])
    x = (m[:, 0] - cm[0]) * sm[0]; y = (m[:, 1] - cm[1]) * sm[1]
    X = (M[:, 0] - cM[0]) * sM[0]; Y = (M[:, 1] - cM[1]) * sM[1]
    o = np.ones(count); z = np.zeros(count)
    Lx = np.stack([X, Y, o, z, z, z, -x * X, -x * Y, -x], 1); Ly = np.stack([z, z, z, X, Y, o, -y * X, -y * Y, -y], 1)
    return Lx.T @ Lx + Ly.T @ Ly, invHnorm, Hnorm2


def run_kernel(a, b):
    """HomographyEstimatorCallback::runKernel: eigenvector of the smallest eigenvalue of L^T L, de-normalised, h22 = 1."""
    r = ltl(a, b)
    if r is None:
        return None
    L, invHnorm, Hnorm2 = r
    _, V = np.linalg.eigh(L)
    H = invHnorm @ V[:, 0].reshape(3, 3) @ Hnorm2
    return H / H[2, 2]


def _residuals(h, M, m, jac):
    Mx = M[:, 0]; My = M[:, 1]
    ww = h[6] * Mx + h[7] * My + 1.0
    ww = np.where(np.abs(ww) > DBL_EPSILON, 1.0 / np.where(ww == 0, 1.0, ww), 0.0)
    xi = (h[0] * Mx + h[1] * My + h[2]) * ww; yi = (h[3] * Mx + h[4] * My + h[5]) * ww
    r = np.stack([xi - m[:, 0], yi - m[:, 1]], 1).reshape(-1)
    if not jac:
        return r
    J = np.zeros((len(M), 2, 8))
    J[:, 0, 0] = Mx * ww; J[:, 0, 1] = My * ww; J[:, 0, 2] = ww; J[:, 0, 6] = -Mx * ww * xi; J[:, 0, 7] = -My * ww * xi
    J[:, 1, 3] = Mx * ww; J[:, 1, 4] = My * ww; J[:, 1, 5] = ww; J[:, 1, 6] = -Mx * ww * yi; J[:, 1, 7] = -My * ww * yi
    return r, J.reshape(-1, 8)


def refine_lm(H, a, b, max_iters=10):
    """LMSolverImpl::run on the 8 parameters h00..h21 (HomographyRefineCallback residuals), eps = FLT_EPSILON."""
    M = np.asarray(a, np.float32).astype(np.float64); m = np.asarray(b, np.float32).astype(np.float64)
    x = np.asarray(H, np.float64).reshape(-1)[:8].copy()
    r, J = _residuals(x, M, m, True)
    S = r @ r; A = J.T @ J; v = J.T @ r; D = np.diag(A).copy()
    lam, lc = 1.0, 0.75
    it = 0
    while True:
        d = np.linalg.solve(A + np.diag(lam * D), v)
        xd = x - d
        rd = _residuals(xd, M, m, False)
        Sd = rd @ rd
        dS = d @ (2 * v - A @ d)
        R = (S - Sd) / (dS if abs(dS) > DBL_EPSILON else 1.0)
        if R > 0.75:
            lam *= 0.5
            if lam < lc:
                lam = 0.0
        elif R < 0.25:
            t = d @ v
            nu = (Sd - S) / (t if abs(t) > DBL_EPSILON else 1.0) + 2
            nu = min(max(nu, 2.0), 10.0)
            if lam == 0:
                maxval = max(DBL_EPSILON, np.abs(np.diag(np.linalg.inv(A))).max())
                lam = lc = 1.0 / maxval
                nu *= 0.5
            lam *= nu
        if Sd < S:
            S = Sd; x = xd
            r, J = _residuals(x, M, m, True)
            A = J.T @ J; v = J.T @ r
        it += 1
        if not (it < max_iters and np.abs(d).max() >= FLT_EPSILON and np.abs(r).max() >= FLT_EPSILON):
            break
    out = np.append(x, 1.0).reshape(3, 3)
    return out / out[2, 2]


def ransac(a, b, threshold=10.0, max_iters=2000, confidence=0.995):
    """The RANSAC phase.  Returns (H or None, mask of H, visited [(quad or None, count or -1)], iterations)."""
    a = np.asarray(a, np.float32).reshape(-1, 2); b = np.asarray(b, np.float32).reshape(-1, 2)
    n = len(a); t2 = np.float32(np.float64(threshold) ** 2)
    rng = CvRng()
    niters = max(max_iters, 1); best = None; best_mask = None; max_good = 0; visited = []
    it = 0
    while it < niters:
        idx = get_subset(a, b, rng)
        if idx is None:
            if it == 0:
                return None, np.zeros(n, np.uint8), visited, 0
            break
        H = run_kernel(a[idx], b[idx])
        g = -1
        if H is not None:
            mask = err_homography(H, a, b) <= t2
            g = int(mask.sum())
            if g > max(max_good, 3):
                best, best_mask, max_good = H, mask, g
                niters = ransac_update_num_iters(confidence, (n - g) / n, 4, niters)
        visited.append((idx, g))
        it += 1
    if best is None:
        return None, np.zeros(n, np.uint8), visited, it
    return best, best_mask.astype(np.uint8), visited, it


def find_homography(a, b, threshold=10.0, max_iters=2000, confidence=0.995, refine_iters=10):
    """cv::findHomography(a, b, RANSAC, threshold, mask, max_iters, confidence).  Returns a dict with H (None when there is no
    model), mask, n_inliers, ransac_H, ransac_mask, ransac_inliers, visited, iterations."""
    a = np.asarray(a, np.float32).reshape(-1, 2); b = np.asarray(b, np.float32).reshape(-1, 2)
    n = len(a); t2 = np.float32(np.float64(threshold) ** 2)
    out = dict(H=None, mask=np.zeros(n, np.uint8), n_inliers=0, ransac_H=None, ransac_mask=np.zeros(n, np.uint8), ransac_inliers=0,
               visited=[], iterations=0)
    if n < 4:
        return out
    if n == 4:                       # findHomography: no RANSAC and no refinement for exactly four points, the mask is all ones
        H = run_kernel(a, b)
        if H is not None:
            ones = np.ones(4, np.uint8)
            out.update(H=H, mask=ones, n_inliers=4, ransac_H=H, ransac_mask=ones, ransac_inliers=4)
        return out
    H, mask, visited, it = ransac(a, b, threshold, max_iters, confidence)
    out.update(visited=visited, iterations=it)
    if H is None:
        return out
    out.update(ransac_H=H, ransac_mask=mask, ransac_inliers=int(mask.sum()))
    sel = mask.astype(bool)
    Hr = run_kernel(a[sel], b[sel])
    if Hr is None:
        Hr = H
    Hr = refine_lm(Hr, a[sel], b[sel], refine_iters)
    fm = (err_homography(Hr, a, b) <= t2).astype(np.uint8)
    out.update(H=Hr, mask=fm, n_inliers=int(fm.sum()))
    return out
