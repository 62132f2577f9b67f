"""Bundle-adjustment fixtures that leave the one path `synth.make_ba_problem` takes (cameras on a circle, equal track lengths,
gentle perturbation, convergence by function tolerance): each edits a `make_ba_problem` output in numpy so that the LM
solver meets rejected steps, clamped LM diagonals, ill-conditioned points, outliers, negative depths, ragged tracks and the
three FAILURE paths.  Shared by test_oracle_ba_lm_paths.py (the oracle against itself and oracle/dense_lm.py) and
test_gpu_ba_lm_paths.py (the GPU against the oracle).

A case is a dict: `args` = (cams, pts, focal, obs_xy, obs_cam, pt_off) in the C ABI layout, `opts` = option overrides that
define the case (for both the GPU and the oracle).
"""
import numpy as np

from sfm_toy_library_b200 import synth


def args_of(p):
    return p["cams"], p["pts"], p["focal"], p["obs_xy"], p["obs_cam"], p["pt_off"]


def _rot(cams):
    return np.stack([synth.angle_axis_to_rotmat(c[:3]) for c in cams])


def project(cams, pts, focal, obs_cam, pt_off):
    """SimpleReprojectionError's prediction (principal point subtracted) of every observation, float64."""
    obs_pt = np.repeat(np.arange(len(pts)), np.diff(pt_off))
    P = np.einsum("oij,oj->oi", _rot(cams)[obs_cam], pts[obs_pt]) + cams[obs_cam, 3:]
    return focal * P[:, :2] / P[:, 2:3], P[:, 2]


def observe(cams_true, pts_true, focal_true, tracks, seed, noise_px=0.5, cam_sigma=(0.01, 0.05), pt_sigma=0.05, f_factor=1.02):
    """A problem from ground truth and per-point camera lists (ascending): noisy float32 observations and a perturbed start."""
    rs = np.random.RandomState(seed)
    obs_cam = np.concatenate([np.asarray(t, np.int32) for t in tracks]) if tracks else np.zeros(0, np.int32)
    pt_off = np.r_[0, np.cumsum([len(t) for t in tracks])].astype(np.int32)
    xy, _ = project(cams_true, pts_true, focal_true, obs_cam, pt_off)
    obs_xy = (xy + rs.normal(0, noise_px, xy.shape)).astype(np.float32)
    nc = len(cams_true)
    cams = cams_true + np.c_[rs.normal(0, cam_sigma[0], (nc, 3)), rs.normal(0, cam_sigma[1], (nc, 3))]
    pts = pts_true + rs.normal(0, pt_sigma, pts_true.shape)
    return dict(args=(cams, pts, focal_true * f_factor, obs_xy, obs_cam.astype(np.int32), pt_off), opts={})


def _centres(cams):
    return -np.einsum("cji,cj->ci", _rot(cams), cams[:, 3:])


# ---------------------------------------------------------------------------------------------------------------- fixtures
def wide(seed=0):
    """Cameras perturbed 30x harder than make_ba_problem (0.3 rad, 1.5 m), points 40x (2 m): 26 LM iterations, 6 of them
    rejected steps.  (10x perturbations converge in five accepted steps.)"""
    p = synth.make_ba_problem(n_cams=6, n_pts=120, obs_per_pt=4, seed=seed)
    cams = p["cams_true"] + 30 * (p["cams"] - p["cams_true"])
    pts = p["pts_true"] + 40 * (p["pts"] - p["pts_true"])
    return dict(args=(cams, pts, p["focal"], p["obs_xy"], p["obs_cam"], p["pt_off"]), opts={})


def far_points(seed=4, share=0.2):
    """A share of the points at depth 1e3..1e5 along the viewing direction of a camera, observed by the cameras that look
    towards them: their Jacobi-scaled columns fall below min_lm_diagonal, so the clamp of the point blocks is active."""
    p = synth.make_ba_problem(n_cams=8, n_pts=100, obs_per_pt=4, seed=seed)
    rs = np.random.RandomState(100 + seed)
    ct, pt = p["cams_true"], p["pts_true"].copy()
    R, ctr = _rot(ct), _centres(ct)
    tracks = [list(p["obs_cam"][p["pt_off"][i]:p["pt_off"][i + 1]]) for i in range(p["np"])]
    for i in rs.choice(p["np"], int(share * p["np"]), replace=False):
        c0 = rs.randint(p["nc"])
        pt[i] = R[c0, 2] * 10 ** rs.uniform(3, 5) + rs.uniform(-1, 1, 3)
        vis = [c for c in range(p["nc"]) if R[c, 2] @ (pt[i] - ctr[c]) > 0.7 * np.linalg.norm(pt[i] - ctr[c])]
        tracks[i] = sorted(rs.choice(vis, min(3, len(vis)), replace=False)) if len(vis) >= 2 else [c0]
    case = observe(ct, pt, p["focal_true"], tracks, seed)
    # f / depth makes their scaled columns 1e-4..1e-2: a min_lm_diagonal of 1e-3 binds on them (and on no near point).  The
    # free solve crawls along the far points' depths for over a hundred iterations, along which two correct solvers'
    # rounding drifts apart (1e-7 in the cost after 40): 12 iterations
    case["opts"] = dict(min_lm_diagonal=1e-3, max_num_iterations=12)
    return case


def short_baseline(seed=5, n_pairs=25):
    """An extra camera 1e-3 from camera 0 with the same orientation, and points seen only by the two of them."""
    p = synth.make_ba_problem(n_cams=6, n_pts=120, obs_per_pt=3, seed=seed)
    rs = np.random.RandomState(200 + seed)
    ct = np.vstack([p["cams_true"], p["cams_true"][:1]])
    ct[-1, 3:] += _rot(ct[:1])[0] @ np.array([1e-3, 0, 0])
    R0, c0 = _rot(ct[:1])[0], _centres(ct[:1])[0]
    extra = c0 + (R0[2] * rs.uniform(8, 12, (n_pairs, 1))) + rs.uniform(-1.5, 1.5, (n_pairs, 3))
    pts = np.vstack([p["pts_true"], extra])
    tracks = [list(p["obs_cam"][p["pt_off"][i]:p["pt_off"][i + 1]]) for i in range(p["np"])] + [[0, 6]] * n_pairs
    case = observe(ct, pts, p["focal_true"], tracks, seed)
    case["opts"] = dict(max_num_iterations=40)      # the free solve takes 138 iterations
    return case


def outliers(seed=6, share=0.05):
    """5 % of the observations moved by 200 px."""
    p = synth.make_ba_problem(n_cams=8, n_pts=200, obs_per_pt=4, seed=seed)
    rs = np.random.RandomState(300 + seed)
    xy = p["obs_xy"].copy()
    idx = rs.choice(p["nobs"], int(share * p["nobs"]), replace=False)
    ang = rs.uniform(0, 2 * np.pi, len(idx))
    xy[idx] += (200 * np.c_[np.cos(ang), np.sin(ang)]).astype(np.float32)
    return dict(args=(p["cams"], p["pts"], p["focal"], xy, p["obs_cam"], p["pt_off"]), opts={})


def behind(seed=7, n_behind=4):
    """A few points behind one of the cameras that observe them (negative depth, finite residual)."""
    p = synth.make_ba_problem(n_cams=8, n_pts=150, obs_per_pt=3, seed=seed)
    rs = np.random.RandomState(400 + seed)
    ct, pt = p["cams_true"], p["pts_true"].copy()
    ctr = _centres(ct)
    tracks = [list(p["obs_cam"][p["pt_off"][i]:p["pt_off"][i + 1]]) for i in range(p["np"])]
    for i in rs.choice(p["np"], n_behind, replace=False):
        c = tracks[i][0]
        pt[i] = ctr[c] * 1.25 + rs.uniform(-0.3, 0.3, 3)          # beyond camera c, seen from the cameras across the circle
    case = observe(ct, pt, p["focal_true"], tracks, seed)
    _, depth = project(ct, pt, p["focal_true"], case["args"][4], case["args"][5])
    assert (depth < 0).sum() >= n_behind
    return case


def ragged(seed=8, n_cams=64):
    """Track lengths 0, 1, 2..16 and 33..60 in one problem.  1-view points keep a definite point block only while the LM
    diagonal is not vanishingly small: the radius is capped at 1e6."""
    p = synth.make_ba_problem(n_cams=n_cams, n_pts=1, obs_per_pt=1, seed=seed)
    rs = np.random.RandomState(500 + seed)
    lens = [0, 0, 1, 1, 1] + list(range(2, 17)) * 6 + list(range(33, 61)) * 2
    rs.shuffle(lens)
    pts = rs.uniform(-2, 2, (len(lens), 3))
    tracks = [sorted(rs.choice(n_cams, k, replace=False)) for k in lens]
    case = observe(p["cams_true"], pts, p["focal_true"], tracks, seed)
    case["opts"] = dict(max_trust_region_radius=1e6)
    return case


def track_lengths(maxk, seed=9, n_pts=None, n_cams=None):
    """Tracks of length 2..maxk, a few of exactly maxk (every G bucket / the staged and unstaged paths)."""
    n_cams = n_cams or max(maxk + 1, 6)
    n_pts = n_pts or 60
    p = synth.make_ba_problem(n_cams=n_cams, n_pts=1, obs_per_pt=1, seed=seed)
    rs = np.random.RandomState(600 + seed)
    lens = np.minimum(maxk, rs.randint(2, maxk + 1, n_pts))
    lens[:3] = maxk
    pts = rs.uniform(-2, 2, (n_pts, 3))
    tracks = [sorted(rs.choice(n_cams, k, replace=False)) for k in lens]
    return observe(p["cams_true"], pts, p["focal_true"], tracks, seed)


def eval_fail(seed=10):
    """One NaN observation: the cost at x0 is not finite."""
    p = synth.make_ba_problem(n_cams=5, n_pts=80, obs_per_pt=3, seed=seed)
    xy = p["obs_xy"].copy(); xy[17, 1] = np.nan
    return dict(args=(p["cams"], p["pts"], p["focal"], xy, p["obs_cam"], p["pt_off"]), opts={})


def chol_fail(seed=11):
    """A camera nobody observes and min_lm_diagonal = 0: its column norms are 0, so its LM diagonal and its whole block of
    the reduced system are exactly zero, and the dense Cholesky fails at every iteration.  Every other column keeps its
    LM diagonal (max_lm_diagonal stays 1e32): with it at 0 too, the undamped gauge directions of the observed cameras
    would make the factor fail everywhere.  Camera 6 of 7 puts the zero rows (36..41 of n = 43) inside the last, padded
    32-row tile, whose factorisation replaces a bad pivot by 1: the factor stays finite and only the Cholesky's failure
    flag makes the step invalid (a zero pivot in an earlier tile would also turn the step into NaN)."""
    p = synth.make_ba_problem(n_cams=7, n_pts=140, obs_per_pt=3, seed=seed)
    keep = np.array([6 not in p["obs_cam"][p["pt_off"][i]:p["pt_off"][i + 1]] for i in range(p["np"])])
    sel = np.repeat(keep, 3)
    off = (np.arange(keep.sum() + 1) * 3).astype(np.int32)
    return dict(args=(p["cams"], p["pts"][keep], p["focal"], p["obs_xy"][sel], p["obs_cam"][sel], off),
                opts=dict(min_lm_diagonal=0.0))


def point_fail(seed=12):
    """focal = 0 and min_lm_diagonal = max_lm_diagonal = 0: every point's Jacobian and LM diagonal, so every point block,
    is exactly zero."""
    p = synth.make_ba_problem(n_cams=5, n_pts=80, obs_per_pt=3, seed=seed)
    return dict(args=(p["cams"], p["pts"], 0.0, p["obs_xy"], p["obs_cam"], p["pt_off"]),
                opts=dict(min_lm_diagonal=0.0, max_lm_diagonal=0.0))


FIXTURES = dict(wide=wide, far_points=far_points, short_baseline=short_baseline, outliers=outliers, behind=behind,
                ragged=ragged, eval_fail=eval_fail, chol_fail=chol_fail, point_fail=point_fail)


# ------------------------------------------------------------------------------------------------------- termination paths
# (fixture, option overrides, termination type, message up to its first number).  Every one is admissible: the oracle takes
# the same decisions with either Jacobian and with 1 or 32 threads (test_oracle_ba_lm_paths.py).
CONVERGENCE, NO_CONVERGENCE, FAILURE = 0, 1, 2
PATHS = {
    "function_tol": ("wide", {}, CONVERGENCE, "Function tolerance reached. |cost_change|/cost: "),
    "gradient_tol": ("wide", dict(gradient_tolerance=10.0), CONVERGENCE, "Gradient tolerance reached."),
    "parameter_tol": ("wide", dict(parameter_tolerance=1e-5, function_tolerance=1e-12), CONVERGENCE,
                      "Parameter tolerance reached. Relative step_norm: "),
    # both stopping tests of an iteration's start hold at once: the first accepted step lands on the radius cap, which is
    # also the minimum radius, at a point whose gradient is below the tolerance; Ceres tests the gradient first
    "gradient_before_min_radius": ("wide", dict(gradient_tolerance=5e6, max_trust_region_radius=5e3, min_trust_region_radius=5e3),
                                   CONVERGENCE, "Gradient tolerance reached."),
    "min_radius": ("behind", dict(min_relative_decrease=0.9999, min_trust_region_radius=1.0), CONVERGENCE,
                   "Minimum trust region radius reached."),
    "max_radius": ("outliers", dict(initial_trust_region_radius=10.0, max_trust_region_radius=40.0), CONVERGENCE,
                   "Function tolerance reached. |cost_change|/cost: "),
    "chol_fail_1": ("chol_fail", dict(max_num_consecutive_invalid_steps=1), FAILURE,
                    "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps: "),
    "chol_fail_3": ("chol_fail", dict(max_num_consecutive_invalid_steps=3), FAILURE,
                    "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps: "),
    "point_fail_1": ("point_fail", dict(max_num_consecutive_invalid_steps=1), FAILURE,
                     "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps: "),
    "point_fail_3": ("point_fail", dict(max_num_consecutive_invalid_steps=3), FAILURE,
                     "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps: "),
    "eval_fail": ("eval_fail", {}, FAILURE, "Residual and Jacobian evaluation failed."),
    # non-default options: no Jacobi scaling, and LM diagonal clamps that bind at both ends (between the quartiles of the
    # column norms at x0, see binding_bounds)
    "no_scaling": ("wide", dict(jacobi_scaling=0), CONVERGENCE, "Function tolerance reached. |cost_change|/cost: "),
    "clamp_both_ends": ("wide", dict(min_lm_diagonal=0.9955, max_lm_diagonal=0.9965), CONVERGENCE,
                        "Function tolerance reached. |cost_change|/cost: "),
    "no_scaling_clamped": ("wide", dict(jacobi_scaling=0, min_lm_diagonal=2e5, max_lm_diagonal=3.5e5), CONVERGENCE,
                           "Function tolerance reached. |cost_change|/cost: "),
    "max_iter_0": ("wide", dict(max_num_iterations=0), NO_CONVERGENCE, "Maximum number of iterations reached."),
    "max_iter_1": ("wide", dict(max_num_iterations=1), NO_CONVERGENCE, "Maximum number of iterations reached."),
}


def path_case(name):
    fx, opts, term, msg = PATHS[name]
    case = FIXTURES[fx]()
    return dict(args=case["args"], opts={**case["opts"], **opts}, termination=term, message=msg)


def binding_bounds(oracle, args, jacobi_scaling):
    """(min_lm_diagonal, max_lm_diagonal) between the quartiles of diag(J^T J) of the (scaled) Jacobian at x, so that the
    clamp binds at both ends.  The squared column norms come from the oracle's Jacobi scale s = 1 / (1 + |col|)."""
    s = oracle.ba_reduced_system(*args, radius=1e4, jacobi_scaling=1)["scale"]
    col = 1.0 / s - 1.0
    colsq = (col * s) ** 2 if jacobi_scaling else col ** 2
    return float(np.quantile(colsq, 0.25)), float(np.quantile(colsq, 0.75))
