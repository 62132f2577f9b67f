"""Two-view DLT null vectors (csrc/dlt_math.cuh) at degenerate geometry: scene builders, the 4 x 4 matrices the kernels build,
an exact reference at 40 digits, and a per-point tolerance that follows the point's own conditioning.

The kernels solve A v = 0 for the unit null vector v of the 4 x 4 DLT matrix A, first in closed form (Newton on the
characteristic polynomial of A^T A, then an adjugate column) and, when one of its gates declines, by one-sided Jacobi.  The
closed-form gate compares a product of eigenvalue gaps with the cube of the trace, so it depends on the world unit: the scenes
here put points on either side of it, and on the degenerate geometry where the true answer is itself ill-conditioned.
"""
import ctypes as C
import os
import subprocess

import mpmath
import numpy as np

from sfm_toy_library_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = synth.TEST_K
U24, U53 = 2.0 ** -24, 2.0 ** -53
FALLBACK_G, FAST_G = 1e-9, 1e-5          # 100x either side of the gate's 1e-7: device FMA contraction cannot flip these
RANK_DEFICIENT = 1e-12                   # sigma3 - sigma4 <= this * sigma1: the null vector is not unique


# ---------------------------------------------------------------- scenes (float32 pixels, float32 poses)
def _pose(R, t):
    return np.c_[np.asarray(R, np.float64), np.asarray(t, np.float64)].astype(np.float32)


def _project(P, X):
    Xc = X @ P[:, :3].astype(np.float64).T + P[:, 3].astype(np.float64)
    return Xc[:, :2] / Xc[:, 2:3]


def _scene(Pl, Pr, X, rs, noise_px=0.2):
    """pixels of X in both views with Gaussian noise, rounded to float32"""
    out = [(_project(P, X) * K[0, 0] + K[:2, 2] + rs.normal(0, noise_px, (len(X), 2))).astype(np.float32) for P in (Pl, Pr)]
    return dict(K=K.copy(), Pl=Pl, Pr=Pr, ptsL=out[0], ptsR=out[1])


def rot(w):
    w = np.asarray(w, np.float64); th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th; Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def fixture_scaled(s, n, seed=0):
    """make_triangulation_problem's scene (the fixture poses, the same point box and noise) with the world unit scaled by s"""
    rs = np.random.RandomState(seed)
    Pl, Pr = synth.fixture_poses()
    Pl = Pl.copy(); Pr = Pr.copy(); Pl[:, 3] *= np.float32(s); Pr[:, 3] *= np.float32(s)
    X = np.stack([rs.uniform(-20, 40, n), rs.uniform(-20, 20, n), rs.uniform(30, 80, n)], 1) * s
    return _scene(Pl, Pr, X, rs, noise_px=0.7)


def offset_scene(off, n, seed=0):
    """the fixture scene (unit scale) moved by off * (1, 0.3, -0.5): the cameras sit `off` units from the world origin"""
    rs = np.random.RandomState(seed)
    Pl0, Pr0 = synth.fixture_poses()
    T = off * np.array([1.0, 0.3, -0.5])
    Pl, Pr = (_pose(P[:, :3], P[:, 3].astype(np.float64) - P[:, :3].astype(np.float64) @ T) for P in (Pl0, Pr0))
    X = np.stack([rs.uniform(-20, 40, n), rs.uniform(-20, 20, n), rs.uniform(30, 80, n)], 1) + T
    return _scene(Pl, Pr, X, rs, noise_px=0.7)


def baseline_scene(b, depth, forward, n, seed=0):
    """[I|0] and a camera turned by 0.01 rad and moved by b sideways or forwards; points at depth/2 .. depth"""
    rs = np.random.RandomState(seed)
    Pl = _pose(np.eye(3), [0, 0, 0]); Pr = _pose(rot([0, 0.01, 0]), [0, 0, -b] if forward else [-b, 0, 0])
    X = np.stack([rs.uniform(-0.3, 0.3, n) * depth, rs.uniform(-0.3, 0.3, n) * depth, rs.uniform(0.5, 1.0, n) * depth], 1)
    return _scene(Pl, Pr, X, rs)


def epipole_scene(r_px, n, seed=0):
    """forward motion by one unit: matches r_px pixels from the epipole (the principal point) in the left view, noise-free"""
    rs = np.random.RandomState(seed)
    Pl = _pose(np.eye(3), [0, 0, 0]); Pr = _pose(np.eye(3), [0, 0, -1])
    ang = rs.uniform(0, 2 * np.pi, n); d = rs.uniform(5, 40, n); rad = r_px / K[0, 0] * d
    return _scene(Pl, Pr, np.c_[rad * np.cos(ang), rad * np.sin(ang), d], rs, noise_px=0.0)


def special_scene(kind, n, seed=0):
    """'rotation': both centres at the origin; 'identical': the same camera twice and the same pixels in both views (A has rank 2,
    so its null vector is not unique); 'behind': points behind both cameras"""
    rs = np.random.RandomState(seed)
    X = np.stack([rs.uniform(-5, 5, n), rs.uniform(-5, 5, n), rs.uniform(10, 30, n)], 1)
    Pl = _pose(np.eye(3), [0, 0, 0])
    if kind == "rotation":
        return _scene(Pl, _pose(rot([0, 0.1, 0]), [0, 0, 0]), X, rs)
    if kind == "identical":
        sc = _scene(Pl, Pl.copy(), X, rs)
        sc["ptsR"] = sc["ptsL"].copy()
        return sc
    assert kind == "behind"
    X[:, 2] *= -1
    return _scene(Pl, _pose(rot([0, 0.05, 0]), [-1, 0, 0]), X, rs)


def sweep():
    """the named scenes of the host and GPU tests: (name, scene)"""
    out = [(f"fixture x{s:g}", fixture_scaled(s, 2000, seed=k)) for k, s in enumerate((1e-4, 1e-2, 1, 4, 8, 10, 100, 1e4))]
    out += [("offset 100", offset_scene(100.0, 2000)), ("offset 1000", offset_scene(1000.0, 2000, seed=1))]
    out += [(f"baseline {b:g} depth {d:g} {'forward' if fw else 'side'}", baseline_scene(b, d, fw, 500, seed=k))
            for k, (b, d, fw) in enumerate((b, d, fw) for b in (1.0, 1e-3, 1e-4, 1e-5) for d in (3.0, 3000.0) for fw in (False, True))]
    out += [(f"epipole {r:g} px", epipole_scene(r, 500, seed=k)) for k, r in enumerate((0.0, 0.01, 0.1, 1.0))]
    out += [(k, special_scene(k, 1000)) for k in ("rotation", "identical", "behind")]
    return out


def subsample(m, cap, seed=0):
    return np.arange(m) if m <= cap else np.sort(np.random.RandomState(seed).choice(m, cap, replace=False))


# ---------------------------------------------------------------- the matrices the kernels build
def triangulation_matrices(K, Pl, Pr, ptsL, ptsR):
    """A [m, 4, 4] of triangulate_kernel: x_n = (u - c) * (1/f) in double rounded to float, rows x P[2] - P[0], y P[2] - P[1]"""
    K = np.asarray(K, np.float32).reshape(3, 3)
    fx, fy, cx, cy = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))

    def norm(p):
        p = np.asarray(p, np.float32).astype(np.float64)
        return (((p[:, 0] - cx) * (1.0 / fx)).astype(np.float32).astype(np.float64),
                ((p[:, 1] - cy) * (1.0 / fy)).astype(np.float32).astype(np.float64))
    (xl, yl), (xr, yr) = norm(ptsL), norm(ptsR)
    PL = np.asarray(Pl, np.float32).astype(np.float64).reshape(3, 4); PR = np.asarray(Pr, np.float32).astype(np.float64).reshape(3, 4)
    return np.ascontiguousarray(np.stack([xl[:, None] * PL[2] - PL[0], yl[:, None] * PL[2] - PL[1],
                                          xr[:, None] * PR[2] - PR[0], yr[:, None] * PR[2] - PR[1]], 1))


def cheirality_matrices(a, b, f, cx, cy, Pc):
    """A [m, 4, 4] of essential_cheirality_kernel for candidate Pc = [R|t] (3 x 4 double): x = (u - c) / f in double"""
    x1 = (np.asarray(a, np.float64) - [cx, cy]) / f; x2 = (np.asarray(b, np.float64) - [cx, cy]) / f
    m = len(x1); A = np.zeros((m, 4, 4))
    A[:, 0, 0] = -1.0; A[:, 0, 2] = x1[:, 0]; A[:, 1, 1] = -1.0; A[:, 1, 2] = x1[:, 1]
    A[:, 2, :] = x2[:, 0:1] * Pc[2] - Pc[0]; A[:, 3, :] = x2[:, 1:2] * Pc[2] - Pc[1]
    return A


# ---------------------------------------------------------------- the host build of dlt_math.cuh
_LIB = None


def host_lib():
    """tests/host_dlt.cpp compiled with g++ (no FMA contraction): the device's null-vector code on the CPU"""
    global _LIB
    if _LIB is None:
        so = os.path.join(ROOT, "tests", "_build", "libhost_dlt.so")
        os.makedirs(os.path.dirname(so), exist_ok=True)
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([cxx, "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_dlt.cpp"),
                        "-o", so], check=True)
        _LIB = C.CDLL(so)
    return _LIB


def host_null_vectors(A):
    """-> (closed-form v [m, 4] (zeros where it declines), accepted [m], Jacobi v [m, 4])"""
    A = np.ascontiguousarray(A, np.float64).reshape(-1, 16)
    m = len(A); vf = np.zeros((m, 4)); ok = np.zeros(m, np.int32); vj = np.zeros((m, 4))
    d = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
    host_lib().host_null_vectors(d(A), m, d(vf), ok.ctypes.data_as(C.POINTER(C.c_int)), d(vj))
    return vf, ok.astype(bool), vj


def dehomogenise(v):
    """the kernel's float dehomogenisation: (float) v[:3] * (1 / (float) v[3]) in float, scale 1 where w == 0"""
    h = np.asarray(v, np.float64).reshape(-1, 4).astype(np.float32)
    w = h[:, 3]
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        sc = np.where(w != 0, np.float32(1) / np.where(w != 0, w, np.float32(1)), np.float32(1)).astype(np.float32)
        return h[:, :3] * sc[:, None]


# ---------------------------------------------------------------- exact reference
def exact(A):
    """per matrix, from the eigen-decomposition of A^T A at 40 digits: singular values sigma [m, 4] (descending), the unit null
    vector v [m, 4] (rounded to double), X* [m, 3] (the kernel's dehomogenisation of v, i.e. the correctly rounded answer) and the
    closed-form gate's margin g = prod_{i<4}(lambda_i - lambda_4) / (trace^3 / 64) [m]"""
    A = np.asarray(A, np.float64).reshape(-1, 4, 4)
    sig = np.zeros((len(A), 4)); v = np.zeros((len(A), 4)); g = np.zeros(len(A))
    with mpmath.workdps(40):
        for k, a in enumerate(A):
            M = mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in a])
            E, Q = mpmath.eigsy(M.T * M)
            order = sorted(range(4), key=lambda i: -E[i])
            lam = [max(E[i], mpmath.mpf(0)) for i in order]
            sig[k] = [float(mpmath.sqrt(x)) for x in lam]
            v[k] = [float(Q[r, order[3]]) for r in range(4)]
            tr = lam[0] + lam[1] + lam[2] + lam[3]
            g[k] = float((lam[0] - lam[3]) * (lam[1] - lam[3]) * (lam[2] - lam[3]) / (tr ** 3 / 64)) if tr > 0 else 0.0
    return dict(sigma=sig, v=v, X=dehomogenise(v).astype(np.float64), g=g)


def error_ratio(X, A, ref):
    """per point, |error| / tolerance (<= 1 passes).
    Unique null vector: delta = 16 u53 sigma1 / (sigma3 - sigma4) bounds the angle error of a backward-stable null vector;
    with n = |(X*, 1)| the tolerance is 8 u24 |X*| + delta n (1 + |X*|).
    Rank-deficient (sigma3 - sigma4 <= 1e-12 sigma1): (X, 1) must lie in the null space, |A (X, 1)| <= 16 u24 sigma1 |(X, 1)|."""
    X = np.asarray(X, np.float64).reshape(-1, 3); A = np.asarray(A, np.float64).reshape(-1, 4, 4)
    s = ref["sigma"]; Xs = ref["X"]
    gap = s[:, 2] - s[:, 3]
    deficient = gap <= RANK_DEFICIENT * s[:, 0]
    nx = np.linalg.norm(Xs, axis=1); n = np.sqrt(1.0 + nx ** 2)
    with np.errstate(divide="ignore", invalid="ignore"):
        delta = 16 * U53 * s[:, 0] / gap
        tol = 8 * U24 * nx + delta * n * (1 + nx)
        r = np.linalg.norm(X - Xs, axis=1) / tol
        Xh = np.c_[X, np.ones(len(X))]
        res = np.linalg.norm(np.einsum("kij,kj->ki", A, Xh), axis=1) / (16 * U24 * s[:, 0] * np.linalg.norm(Xh, axis=1))
    r = np.where(deficient, res, r)
    return np.where(np.isfinite(r), r, np.where(np.all(X == Xs, axis=1), 0.0, np.inf))


def path(ref, accepted):
    """'fallback' where the gate margin is <= 1e-9, 'fast' where it is >= 1e-5 and the host build accepts, '' in between"""
    g = ref["g"] if isinstance(ref, dict) else ref
    return np.where(g <= FALLBACK_G, "fallback", np.where((g >= FAST_G) & accepted, "fast", ""))


def gate_margin(A):
    """g of exact() in double (eigvalsh of A^T A): enough to sort whole scenes by path, far from the 1e-9 / 1e-5 cuts"""
    A = np.asarray(A, np.float64).reshape(-1, 4, 4)
    lam = np.linalg.eigvalsh(np.einsum("kji,kjl->kil", A, A))[:, ::-1]
    tr = lam.sum(1)
    return (lam[:, 0] - lam[:, 3]) * (lam[:, 1] - lam[:, 3]) * (lam[:, 2] - lam[:, 3]) / (tr ** 3 / 64)
