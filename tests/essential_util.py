"""Shared inputs of the essential-matrix tests: five-point samples from the crazyhorse pairs and from a synthetic two-view
scene, the canonical form of a solution, and the constraint residuals of an essential matrix."""
import numpy as np

F, CX, CY = 2500.0, 512.0, 384.0       # the fixture's K


def canon(e):
    """unit Frobenius norm, largest-magnitude entry positive"""
    e = np.asarray(e, np.float64).reshape(-1)
    e = e / np.linalg.norm(e)
    return e * np.sign(e[np.argmax(np.abs(e))])


def constraint_residual(E):
    """max |det E|, |2 E E^T E - tr(E E^T) E| of E scaled to unit norm"""
    E = np.asarray(E, np.float64).reshape(3, 3)
    E = E / np.linalg.norm(E)
    return max(abs(np.linalg.det(E)), np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max())


def epipolar_residual(E, x1, x2):
    E = np.asarray(E, np.float64).reshape(3, 3)
    E = E / np.linalg.norm(E)
    h1 = np.c_[x1, np.ones(len(x1))]; h2 = np.c_[x2, np.ones(len(x2))]
    return np.abs(np.einsum("ij,jk,ik->i", h2, E, h1)).max()


def rot(w):
    w = np.asarray(w, np.float64); th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th; Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def synthetic_scene(seed, n, noise_px=0.0, outliers=0.0, f=F, cx=CX, cy=CY):
    """Points in front of two cameras P0 = [I|0], P1 = [R|t] (|t| = 1), at depths 3..10 over a wide field of view (a
    minimal-sample estimate is then accurate to a few hundredths of a degree at 0.5 px noise); pixel coordinates (float32)
    in both views.  Returns (a, b, R, t, is_outlier)."""
    rs = np.random.RandomState(seed)
    R = rot(rs.normal(0, 0.15, 3))
    t = rs.normal(0, 1, 3); t[2] *= 0.3; t /= np.linalg.norm(t)
    X = np.c_[rs.uniform(-10, 10, n), rs.uniform(-7.5, 7.5, n), rs.uniform(3, 10, n)]
    X2 = X @ R.T + t
    a = np.c_[f * X[:, 0] / X[:, 2] + cx, f * X[:, 1] / X[:, 2] + cy]
    b = np.c_[f * X2[:, 0] / X2[:, 2] + cx, f * X2[:, 1] / X2[:, 2] + cy]
    a += rs.normal(0, noise_px, a.shape); b += rs.normal(0, noise_px, b.shape)
    out = rs.rand(n) < outliers
    b[out] = np.c_[rs.uniform(0, 2 * cx, out.sum()), rs.uniform(0, 2 * cy, out.sum())]
    return a.astype(np.float32), b.astype(np.float32), R, t, out


def five_point_samples(cfg1, n_fixture=500, n_synth=500, seed=0):
    """(x1, x2 [n, 5, 2] normalised coordinates, pixel a, b [n, 5, 2]) from the 21 crazyhorse pairs and a synthetic scene"""
    rs = np.random.RandomState(seed)
    A, B = [], []
    for k in range(n_fixture):
        p = k % len(cfg1.pairs)
        i, j = cfg1.pairs[p]; q, t, _ = cfg1.matches[p]
        idx = rs.choice(len(q), 5, replace=False)
        A.append(cfg1.features[i].points[q][idx]); B.append(cfg1.features[j].points[t][idx])
    a, b, *_ = synthetic_scene(seed + 1, 2000)
    for k in range(n_synth):
        idx = rs.choice(len(a), 5, replace=False)
        A.append(a[idx]); B.append(b[idx])
    A = np.array(A, np.float32); B = np.array(B, np.float32)
    c = np.array([CX, CY])
    return (A.astype(np.float64) - c) / F, (B.astype(np.float64) - c) / F, A, B


def compare_with_cv2(cv2, x1, x2, A, B, E, nsol):
    """The acceptance of a five-point solver against cv2.findEssentialMat on exactly the same 5 points.  Returns
    (fraction of samples with cv2's solution count, cv2 solutions without a match in samples of equal count, worst residuals)."""
    same = 0; unmatched = 0; worst_epi = 0.0; worst_con = 0.0
    for s in range(len(x1)):
        Ec, _ = cv2.findEssentialMat(A[s].astype(np.float64), B[s].astype(np.float64), F, (CX, CY), cv2.RANSAC, 0.999, 1.0)
        nc = 0 if Ec is None else Ec.shape[0] // 3
        ours = [canon(E[s, k]) for k in range(nsol[s])]
        same += nc == nsol[s]
        for e in ours:
            worst_epi = max(worst_epi, epipolar_residual(e, x1[s], x2[s]))
            worst_con = max(worst_con, constraint_residual(e))
        for k in range(nc):
            ec = Ec[3 * k:3 * k + 3]
            # cv2's own solution is off the essential-matrix variety by rho on ill-conditioned samples; it is then held to
            # 1e4 rho (ours satisfy the constraints to rounding level, checked above)
            tol = max(1e-6, 1e4 * constraint_residual(ec))
            d = min([np.abs(e - canon(ec)).max() for e in ours] or [np.inf])
            unmatched += d > tol and nc == nsol[s]
    return same / len(x1), unmatched, worst_epi, worst_con
