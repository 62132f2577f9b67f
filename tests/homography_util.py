"""Shared inputs of the homography RANSAC tests: the crazyhorse pairs of the cfg1 fixture and seeded synthetic planar scenes."""
import numpy as np


def crazyhorse_pairs(cfg):
    """[(a, b)] float32 aligned points of the 21 pairs."""
    out = []
    for p, (i, j) in enumerate(cfg.pairs):
        q, t, _ = cfg.matches[p]
        out.append((np.ascontiguousarray(cfg.features[i].points[q], np.float32), np.ascontiguousarray(cfg.features[j].points[t], np.float32)))
    return out


def planar_scene(seed, n, outlier_ratio, noise=0.5, size=(1024, 768)):
    """n correspondences of a random plane-induced homography, pixel noise on the inliers, uniform outliers."""
    rs = np.random.RandomState(seed)
    w, h = size
    H = np.eye(3) + np.r_[rs.normal(0, 0.08, 6), rs.normal(0, 1e-4, 2), 0].reshape(3, 3)
    H[0, 2] += rs.uniform(-60, 60); H[1, 2] += rs.uniform(-60, 60)
    a = np.c_[rs.uniform(0, w, n), rs.uniform(0, h, n)]
    ph = np.c_[a, np.ones(n)] @ H.T
    b = ph[:, :2] / ph[:, 2:] + rs.normal(0, noise, (n, 2))
    k = int(round(outlier_ratio * n))
    out = rs.choice(n, k, replace=False)
    b[out] = np.c_[rs.uniform(0, w, k), rs.uniform(0, h, k)]
    return a.astype(np.float32), b.astype(np.float32)


def synthetic_scenes():
    """[(name, a, b)]: planar scenes at 0-70 % outliers and 4-5000 matches, plus the degenerate cases."""
    scenes = []
    for s, (n, r) in enumerate([(4, 0.0), (5, 0.0), (6, 0.2), (8, 0.0), (12, 0.3), (30, 0.5), (60, 0.0), (100, 0.1), (200, 0.3), (300, 0.7),
                                (450, 0.5), (700, 0.4), (900, 0.6), (1200, 0.3), (2000, 0.2), (3000, 0.5), (5000, 0.05), (5000, 0.7)]):
        a, b = planar_scene(100 + s, n, r)
        scenes.append((f"planar_n{n}_out{int(r * 100)}", a, b))
    rs = np.random.RandomState(7)
    t = rs.uniform(0, 500, 50)
    line = np.c_[t, 0.5 * t + 10].astype(np.float32)
    scenes.append(("collinear", line, (line * 1.1 + 3).astype(np.float32)))
    same = np.tile(np.array([[100.0, 200.0]], np.float32), (40, 1))
    scenes.append(("identical", same, same + np.float32(5)))
    a, b = planar_scene(300, 4, 0.0)
    scenes.append(("n4_collinear", np.array([[0, 0], [1, 1], [2, 2], [3, 3]], np.float32), b))
    a, b = planar_scene(301, 200, 0.3)
    a[:20] = a[0]; b[:20] = b[0]                # many repeated correspondences
    scenes.append(("repeated", a, b))
    return scenes
