"""The EPnP solver and rotation conversion of csrc/pose_math.cuh and the sequential RANSAC selection of csrc/ransac_select.cuh
(__host__ __device__) compiled with g++ and checked without a GPU: EPnP against exact poses and against cv2.solvePnP(SOLVEPNP_EPNP)
on samples of the crazyhorse PnP sets, degenerate samples, and the selection loop against the restatement of OpenCV's
(tests/essential_oracle.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from cfg1_util import Cfg1
import essential_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _i(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


@pytest.fixture(scope="module")
def hp():
    so = os.path.join(ROOT, "tests", "_build", "libhost_pose.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_pose.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    L.host_update_num_iters.restype = C.c_int
    L.host_update_num_iters.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int]
    return L


def epnp(hp, X, uv, K):
    X = np.ascontiguousarray(X, np.float64).reshape(-1, 5, 3); uv = np.ascontiguousarray(uv, np.float64).reshape(-1, 5, 2)
    ns = len(X); Rt = np.zeros((ns, 12)); ok = np.zeros(ns, np.int32)
    k = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], np.float64)
    hp.host_epnp(_d(X), _d(uv), _d(k), ns, _d(Rt), _i(ok))
    return Rt.reshape(ns, 3, 4), ok


def rot(w):
    R, _ = cv2.Rodrigues(np.asarray(w, np.float64).reshape(3, 1))
    return R


def project(K, R, t, X):
    p = X @ R.T + t
    return (p[:, :2] / p[:, 2:]) * [K[0, 0], K[1, 1]] + [K[0, 2], K[1, 2]]


def pnp_K(cfg, k):
    """The intrinsics of PnP call k: the replay refines the focal length in the bundle adjustment that precedes it."""
    return np.asarray(cfg.g[f"ba_{k}_K_after"], np.float64)


def test_epnp_recovers_exact_pose(hp):
    rs = np.random.RandomState(0)
    K = np.array([[2500.0, 0, 512], [0, 2400.0, 384], [0, 0, 1]])
    Xs, uvs, poses = [], [], []
    for _ in range(300):
        R = rot(rs.normal(0, 0.6, 3)); t = rs.normal(0, 1, 3) + [0, 0, rs.uniform(4, 20)]
        Xc = np.c_[rs.uniform(-2, 2, (5, 2)), rs.uniform(2, 8, 5)]        # in front of the camera
        X = (Xc - t) @ R                                                    # world points
        Xs.append(X); uvs.append(project(K, R, t, X)); poses.append(np.c_[R, t])
    Rt, ok = epnp(hp, np.array(Xs), np.array(uvs), K)
    assert ok.all()
    poses = np.array(poses)
    rel = np.abs(Rt - poses).max(axis=(1, 2)) / np.abs(poses).max(axis=(1, 2))
    assert rel.max() < 1e-9, rel.max()


def test_epnp_on_crazyhorse_samples_matches_cv2(hp):
    cfg = Cfg1()
    rs = np.random.RandomState(1)
    for k in range(cfg.n_pnp):
        X = cfg.g[f"pnp_{k}_p3"].astype(np.float64); uv = cfg.g[f"pnp_{k}_p2"].astype(np.float64); K = pnp_K(cfg, k)
        # EPnP on 5 noisy points is ill-conditioned (M^T M has a 2-dimensional null space whose basis each solver picks its own
        # way), so single samples differ; the distributions agree: 2000 samples per set bring the medians within 1 %
        idx = np.array([rs.choice(len(X), 5, replace=False) for _ in range(2000)])
        Rt, ok = epnp(hp, X[idx], uv[idx], K)
        ours, theirs = [], []
        for s in range(len(idx)):
            okc, rv, tv = cv2.solvePnP(X[idx[s]], uv[idx[s]], K, None, flags=cv2.SOLVEPNP_EPNP)
            if not ok[s] or not okc:
                continue
            ours.append(np.linalg.norm(project(K, Rt[s, :, :3], Rt[s, :, 3], X[idx[s]]) - uv[idx[s]], axis=1).mean())
            theirs.append(np.linalg.norm(project(K, rot(rv), tv.ravel(), X[idx[s]]) - uv[idx[s]], axis=1).mean())
        assert len(ours) >= 1980, (k, len(ours))
        mo, mc = np.median(ours), np.median(theirs)
        assert abs(mo - mc) <= 0.01 * mc, (k, mo, mc)
        assert np.all(np.isfinite(Rt))


def test_degenerate_samples_give_no_pose_and_no_nan(hp):
    K = np.array([[700.0, 0, 320], [0, 700.0, 240], [0, 0, 1]])
    rs = np.random.RandomState(2)
    uv = rs.uniform(0, 600, (5, 2))
    base = rs.normal(0, 1, (5, 3)) + [0, 0, 10]
    cases = {
        "coincident": np.tile([[1.0, 2.0, 10.0]], (5, 1)),
        "collinear": np.outer(np.linspace(-1, 1, 5), [1.0, 2.0, 0.5]) + [0, 0, 10],
        "coplanar": np.c_[rs.normal(0, 1, (5, 2)), np.full(5, 10.0)] @ rot([0.3, -0.2, 0.1]).T,
        "repeated": base[[0, 1, 2, 2, 2]],
        "nan_point": np.where(np.arange(15).reshape(5, 3) == 7, np.nan, base),
        "inf_point": np.where(np.arange(15).reshape(5, 3) == 4, np.inf, base),
    }
    for name, X in cases.items():
        Rt, ok = epnp(hp, X[None], uv[None], K)
        assert ok[0] == 0, name
        assert np.all(Rt == 0), name
    uvn = uv.copy(); uvn[3, 1] = np.nan
    Rt, ok = epnp(hp, base[None], uvn[None], K)
    assert ok[0] == 0 and np.all(np.isfinite(Rt))


def test_rotmat_to_angle_axis_matches_rodrigues(hp):
    rs = np.random.RandomState(3)
    ws = [rs.normal(0, 1, 3) for _ in range(100)]
    axes = [v / np.linalg.norm(v) for v in rs.normal(0, 1, (10, 3))]
    ws += [a * ang for a in axes for ang in (0.0, 1e-9, 1e-4, np.pi - 1e-6, np.pi - 1e-3)]
    for w in ws:
        R = np.ascontiguousarray(rot(w)); out = np.zeros(3)
        hp.host_rotmat_to_aa(_d(R), _d(out))
        assert np.abs(rot(out) - R).max() < 1e-12, (w, out)
        if np.linalg.norm(w) < np.pi - 1e-2:
            assert np.abs(out - w).max() < 1e-12, (w, out)


def _select(hp, nsol, counts, slots, n, max_iters, confidence, model_points):
    nsol = np.ascontiguousarray(nsol, np.int32); counts = np.ascontiguousarray(counts, np.int32); out = np.zeros(3, np.int32)
    hp.host_select(_i(nsol), _i(counts), len(nsol), slots, n, max_iters, C.c_double(confidence), model_points, _i(out))
    return tuple(int(v) for v in out)


def test_selection_matches_sequential_select_pose(hp):
    """One pose per sample (nsol 0 or 1), model_points = 5, max_iters = 100, confidence = 0.99: the PnP RANSAC's parameters."""
    rs = np.random.RandomState(4)
    seqs = [([1, 1, 0, 1, 1], [3, 7, -1, 7, 9], 40),                   # 3 is not > 4; the tie at 7 keeps the first
            ([1] * 100, [4] * 100, 30),                                  # nothing above 4: no model, all 100 samples visited
            ([1] * 100, [30] + [2] * 99, 30),                            # everything an inlier: the budget drops to 0
            ([0] * 100, [-1] * 100, 30)]                                 # no sample gave a pose
    for _ in range(200):
        S = rs.randint(1, 101); n = rs.randint(5, 700)
        ns = (rs.uniform(size=S) > 0.1).astype(np.int32)
        c = np.where(ns == 1, rs.randint(0, n + 1, S), -1)
        seqs.append((ns, c, n))
    for ns, c, n in seqs:
        ns = np.asarray(ns, np.int32); c = np.asarray(c, np.int32)
        ours = _select(hp, ns, c, 1, n, 100, 0.99, 5)
        compact = c[ns == 1]
        best, good, it = eo.sequential_select(ns, compact, n, max_iters=100, confidence=0.99, model_points=5)
        slot = -1 if best < 0 else int(np.flatnonzero(ns == 1)[best])
        assert ours == (slot, good, it), (ns, c, n, ours, (slot, good, it))


def test_selection_matches_sequential_select_essential(hp):
    """Up to 10 solutions per sample in slots of 10, the essential-matrix RANSAC's layout and parameters."""
    rs = np.random.RandomState(5)
    for _ in range(100):
        S = rs.randint(1, 300); n = rs.randint(5, 2000)
        ns = rs.randint(0, 11, S).astype(np.int32)
        padded = np.zeros((S, 10), np.int32)
        for s in range(S):
            padded[s, :ns[s]] = rs.randint(0, n + 1, ns[s])
        ours = _select(hp, ns, padded.ravel(), 10, n, 1000, 0.999, 5)
        compact = np.concatenate([padded[s, :ns[s]] for s in range(S)])
        best, good, it = eo.sequential_select(ns, compact, n, max_iters=1000, confidence=0.999, model_points=5)
        off = np.r_[0, np.cumsum(ns)]
        slot = -1 if best < 0 else int(10 * (np.searchsorted(off, best, side="right") - 1) + best - off[np.searchsorted(off, best, side="right") - 1])
        assert ours == (slot, good, it)


def test_update_num_iters_matches_oracle(hp):
    rs = np.random.RandomState(6)
    for _ in range(2000):
        p = rs.choice([0.99, 0.999, 0.995, 1.0, 0.5]); ep = rs.uniform(-0.1, 1.1); mp = rs.choice([4, 5]); mi = rs.randint(1, 3000)
        assert hp.host_update_num_iters(p, ep, int(mp), mi) == eo.ransac_update_num_iters(p, ep, int(mp), mi)
