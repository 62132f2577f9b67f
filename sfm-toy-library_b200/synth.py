"""Synthetic workloads for BASELINE.json configs 2-5 (definitions: SURVEY.md section 8(d)).

Shared by tests/ and bench.py.  Pure numpy, deterministic in the seed; nothing here touches the GPU.
"""
import numpy as np


# ------------------------------------------------------------------ small rotation helpers (double)
def euler_deg_to_rotmat(pitch, roll, yaw):
    """ceres::EulerAnglesToRotationMatrix(euler, 3, R): R = Rz(yaw) * Ry(roll) * Rx(pitch), degrees, row-major
    (used by the reference's test fixtures, SfMUnitTests.cpp:85, :121, :135)."""
    p, r, y = np.deg2rad([pitch, roll, yaw])
    c1, s1, c2, s2, c3, s3 = np.cos(y), np.sin(y), np.cos(r), np.sin(r), np.cos(p), np.sin(p)
    return np.array([[c1 * c2, -s1 * c3 + c1 * s2 * s3, s1 * s3 + c1 * s2 * c3],
                     [s1 * c2, c1 * c3 + s1 * s2 * s3, -c1 * s3 + s1 * s2 * c3],
                     [-s2, c2 * s3, c2 * c3]])


def rotmat_to_angle_axis(R):
    R = np.asarray(R, np.float64)
    c = np.clip((np.trace(R) - 1.0) * 0.5, -1.0, 1.0)
    theta = np.arccos(c)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = np.linalg.norm(v) * 0.5
    if s < 1e-12:
        return np.zeros(3) if c > 0 else np.array([np.pi, 0.0, 0.0])
    return v / (2.0 * s) * theta


def angle_axis_to_rotmat(w):
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w)
    if th < 1e-300:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


# ------------------------------------------------------------------ bundle adjustment (configs 2, 3)
def make_ba_problem(n_cams=20, n_pts=10_000, obs_per_pt=8, seed=0, point_seed=None, focal=2500.0,
                    noise_px=0.5, perturb=True):
    """Synthetic BA problem in the flattened layout of the C ABI (include/sfmb200.h):
      cams6 [nc,6] (angle-axis, t) world->camera, pts [np,3], focal, obs_xy [nobs,2] float32 (principal point
      already subtracted, as adjustBundle does at SfMBundleAdjustmentUtils.cpp:149-153), obs_cam [nobs] int32,
      pt_off [np+1] int32; observations sorted by point, then ascending camera (std::map order, :146).
    `seed` fixes the cameras (and the perturbation of cameras/focal); `point_seed` (default: seed) the points,
    so that multi-GPU shards can share cameras but own different points.
    Returns a dict with the initial guess (cams, pts, focal), the ground truth and the observations.
    """
    rs_c = np.random.RandomState(seed)
    ang = np.sort(rs_c.uniform(0, 2 * np.pi, n_cams))
    ctr = np.stack([10 * np.cos(ang), rs_c.uniform(-1, 1, n_cams), 10 * np.sin(ang)], 1)
    cams_true = np.zeros((n_cams, 6))
    Rs = np.zeros((n_cams, 3, 3))
    for i in range(n_cams):
        z = -ctr[i] / np.linalg.norm(ctr[i])
        x = np.cross([0.0, 1.0, 0.0], z); x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z])
        Rs[i] = R
        cams_true[i, :3] = rotmat_to_angle_axis(R)
        cams_true[i, 3:] = -R @ ctr[i]
    cam_noise = np.concatenate([rs_c.normal(0, 0.01, (n_cams, 3)), rs_c.normal(0, 0.05, (n_cams, 3))], 1)

    rs_p = np.random.RandomState(seed if point_seed is None else point_seed)
    pts_true = rs_p.uniform(-2, 2, (n_pts, 3))
    k = min(obs_per_pt, n_cams)
    sel = np.argpartition(rs_p.rand(n_pts, n_cams), k - 1, axis=1)[:, :k]
    sel.sort(axis=1)
    obs_cam = sel.reshape(-1).astype(np.int32)
    obs_pt = np.repeat(np.arange(n_pts), k)
    pt_off = (np.arange(n_pts + 1) * k).astype(np.int32)
    Pc = np.einsum("oij,oj->oi", Rs[obs_cam], pts_true[obs_pt]) + cams_true[obs_cam, 3:]
    proj = focal * Pc[:, :2] / Pc[:, 2:3]
    obs_xy = (proj + rs_p.normal(0, noise_px, proj.shape)).astype(np.float32)
    pt_noise = rs_p.normal(0, 0.05, (n_pts, 3))

    cams0, pts0, f0 = cams_true.copy(), pts_true.copy(), focal
    if perturb:
        cams0 = cams_true + cam_noise
        pts0 = pts_true + pt_noise
        f0 = focal * 1.02
    return dict(nc=n_cams, np=n_pts, nobs=obs_cam.shape[0], cams=cams0, pts=pts0, focal=float(f0),
                cams_true=cams_true, pts_true=pts_true, focal_true=float(focal),
                obs_xy=obs_xy, obs_cam=obs_cam, pt_off=pt_off, obs_pt=obs_pt.astype(np.int32))


BA_CONFIGS = {
    "cfg2": dict(n_cams=20, n_pts=10_000, obs_per_pt=8),      # BASELINE.json configs[1]
    "cfg3": dict(n_cams=100, n_pts=200_000, obs_per_pt=8),    # BASELINE.json configs[2]
}


# ------------------------------------------------------------------ matching (config 4, reference-faithful Hamming)
def make_descriptors(image_id, n=5000, nbytes=32, prev=None, copy_frac=0.2, max_flips=16, n_dups=4):
    """ORB-like 256-bit descriptors: random rows; `copy_frac` of them copied from `prev` (the "previous image")
    with <= max_flips random bit flips so the ratio test passes a realistic share; a few exact duplicate rows
    (tie-break coverage: ties must go to the lower trainIdx)."""
    rs = np.random.RandomState(1000 + image_id)
    d = rs.randint(0, 256, (n, nbytes), dtype=np.uint8)
    if prev is not None and n > 0 and prev.shape[0] > 0:
        m = int(copy_frac * n)
        dst = rs.choice(n, m, replace=False)
        src = rs.randint(0, prev.shape[0], m)
        rows = prev[src].copy()
        for r in range(m):
            nf = rs.randint(0, max_flips + 1)
            bits = rs.randint(0, nbytes * 8, nf)
            for b in bits:
                rows[r, b >> 3] ^= np.uint8(1 << (b & 7))
        d[dst] = rows
    for _ in range(min(n_dups, n // 2)):
        a, b = rs.randint(0, n, 2)
        d[a] = d[b]
    return d


def make_descriptor_set(n_images, n=5000, nbytes=32):
    out, prev = [], None
    for i in range(n_images):
        prev = make_descriptors(i, n, nbytes, prev)
        out.append(prev)
    return out


def make_sift_like(image_id, n=5000, dim=128, prev=None, copy_frac=0.2):
    """Integer-valued float32 SIFT-like descriptors (real SIFT from OpenCV is integer valued, 0..255)."""
    rs = np.random.RandomState(2000 + image_id)
    d = np.minimum(rs.exponential(25.0, (n, dim)), 255).astype(np.int32)
    if prev is not None:
        m = int(copy_frac * n)
        dst = rs.choice(n, m, replace=False); src = rs.randint(0, prev.shape[0], m)
        d[dst] = np.clip(prev[src].astype(np.int32) + rs.randint(-3, 4, (m, dim)), 0, 255)
    return d.astype(np.float32)


# ------------------------------------------------------------------ triangulation (config 5)
TEST_K = np.array([[700.0, 0, 320.0], [0, 700.0, 240.0], [0, 0, 1.0]], np.float32)   # SfMUnitTests.cpp:53-56


def fixture_poses():
    """The reference's stereo fixture (SfMUnitTests.cpp:105-146): float32 3x4 poses."""
    Pl = np.zeros((3, 4), np.float32); Pr = np.zeros((3, 4), np.float32)
    Pl[:, :3] = euler_deg_to_rotmat(5, 5, 5).astype(np.float32); Pl[:, 3] = (-10, 0, 30)
    Pr[:, :3] = euler_deg_to_rotmat(-5, 0, 5).astype(np.float32); Pr[:, 3] = (10, 0, 28)
    return Pl, Pr


CANNED_POINTS = np.array([[4, 12, 50], [12, 11, 55], [22, 1, 45], [13, 3, 60], [11, 16, 61], [21, 12, 65], [24, 11, 67],
                          [29, 6, 41], [27, 4, 44], [22, 7, 58], [20, 9, 51], [15, 10, 40]], np.float32)  # SfMUnitTests.cpp:59-71


def make_triangulation_problem(m=1_000_000, seed=0, noise=1e-3, outlier_frac=0.02):
    """Two fixed cameras (fixture poses), X ~ U([-20,40]x[-20,20]x[30,80]), projected, noise in normalised coords,
    float32 pixels.  A small share of gross outliers exercises the 10 px reprojection filter."""
    rs = np.random.RandomState(seed)
    Pl, Pr = fixture_poses()
    X = np.stack([rs.uniform(-20, 40, m), rs.uniform(-20, 20, m), rs.uniform(30, 80, m)], 1)
    out = []
    for P in (Pl, Pr):
        Xc = X @ P[:, :3].astype(np.float64).T + P[:, 3].astype(np.float64)
        xn = Xc[:, :2] / Xc[:, 2:3] + rs.normal(0, noise, (m, 2))
        out.append((xn * 700.0 + np.array([320.0, 240.0])).astype(np.float32))
    nb = int(outlier_frac * m)
    if nb:
        idx = rs.choice(m, nb, replace=False)
        out[1][idx] += rs.uniform(-60, 60, (nb, 2)).astype(np.float32)
    return dict(K=TEST_K.copy(), Pl=Pl, Pr=Pr, ptsL=out[0], ptsR=out[1], X_true=X.astype(np.float32))


def make_triangulation_pairs(images=50, seed=0):
    """All i < j pairs of `images` views in the layout of sfmb200_triangulate_pairs: pair k is make_triangulation_problem(m, seed
    = 100000 * seed + k) with 400-1200 matches, its two views swapped for odd k, so the pairs alternate between two sets of poses.
    Each pair's key points are appended to its two images.
    Returns (K, poses [P, 2, 3, 4], points per image, pairs [P, 2], match_q, match_t, match_off [P + 1])."""
    rs = np.random.RandomState(seed)
    pts = [[] for _ in range(images)]; sizes = [0] * images
    pairs, poses, mq, mt, off = [], [], [], [], [0]
    for i in range(images):
        for j in range(i + 1, images):
            k = len(pairs); m = int(rs.randint(400, 1201))
            pr = make_triangulation_problem(m, seed=100000 * seed + k)
            (Pl, a), (Pr, b) = ((pr["Pl"], pr["ptsL"]), (pr["Pr"], pr["ptsR"]))[::1 if k % 2 == 0 else -1]
            pts[i].append(a); pts[j].append(b)
            mq.append(np.arange(m, dtype=np.int32) + sizes[i]); mt.append(np.arange(m, dtype=np.int32) + sizes[j])
            sizes[i] += m; sizes[j] += m
            pairs.append((i, j)); poses.append((Pl, Pr)); off.append(off[-1] + m)
    return (TEST_K.copy(), np.array(poses, np.float32), [np.concatenate(p) if p else np.zeros((0, 2), np.float32) for p in pts],
            np.array(pairs, np.int32).reshape(-1, 2), np.concatenate(mq) if mq else np.zeros(0, np.int32),
            np.concatenate(mt) if mt else np.zeros(0, np.int32), np.array(off, np.int64))
