"""The oracle's LM (oracle/ba_oracle.c) on the fixtures of tests/ba_cases.py: rejected steps, clamped LM diagonals, outliers,
negative depths, ragged tracks, and every termination path including the three FAILURE paths.

* Admissibility: the oracle takes exactly the same decisions (termination, iteration count, accept/reject sequence, message
  up to its numbers) with either Jacobian (dual numbers / closed form) and with 1 or 32 threads.  A case whose decisions
  depended on round-off could not be used to hold the GPU to the oracle's decisions; test_gpu_ba_lm_paths.py uses these.
* The oracle against oracle/dense_lm.py (explicit dense Jacobian, full normal equations) wherever dense_lm has the options,
  which pins the reference the GPU is held to on the new branches too.
"""
import re

import numpy as np
import pytest

import ba_cases as bc
from oracle import dense_lm

ALL = [("fixture", n) for n in bc.FIXTURES] + [("path", n) for n in bc.PATHS]


def _case(kind, name):
    return bc.FIXTURES[name]() if kind == "fixture" else bc.path_case(name)


def _solve(oracle, case, **kw):
    o = oracle.ba_default_options(max_solver_time_in_seconds=0.0, **{**case["opts"], **kw})
    return oracle.ba_solve(*case["args"], o, want_trace=True)


def message_prefix(msg):
    """A termination message up to its first number."""
    return re.split(r"[-+]?\d", msg, maxsplit=1)[0]


def decisions(s, trace):
    return (s["termination_type"], s["num_iterations"], s["num_successful_steps"], s["num_unsuccessful_steps"],
            tuple(trace[1:, 2].astype(int)), message_prefix(s["message"]))


@pytest.mark.parametrize("kind,name", ALL, ids=[n for _, n in ALL])
def test_decisions_do_not_depend_on_round_off(oracle, kind, name):
    case = _case(kind, name)
    out = {(mode, nt): decisions(*_solve(oracle, case, jacobian_mode=mode, num_threads=nt)[3:]) for mode in (0, 1) for nt in (1, 32)}
    first = out[(0, 1)]
    for k, d in out.items():
        assert d == first, (k, d, first)
    if kind == "path":
        assert (first[0], first[5]) == (case["termination"], case["message"]), first
    if name in ("wide", "function_tol"):
        assert first[3] >= 5                                      # the point of the fixture: rejected steps
    if name == "gradient_before_min_radius":                      # both tests hold at the check that stops the solve
        c, q, f, s, tr = _solve(oracle, case)
        assert tr[-1, 2] == 1 and tr[-1, 3] <= case["opts"]["gradient_tolerance"] and tr[-1, 1] <= case["opts"]["min_trust_region_radius"]
        assert (tr[:-1, 1] > case["opts"]["min_trust_region_radius"]).all()
    if name == "max_radius":
        tr = _solve(oracle, case)[4]
        assert (tr[1:, 1] == case["opts"]["max_trust_region_radius"]).sum() >= 3   # the cap binds, repeatedly


def test_far_points_clamp_the_point_diagonal(oracle):
    """The fixture's point: the scaled column norms of some point coordinates are below its min_lm_diagonal."""
    case = bc.far_points()
    cams, pts, f, xy, cam, off = case["args"]
    o = oracle.ba_reduced_system(cams, pts, f, xy, cam, off, radius=1e4)
    Jsq = np.zeros(len(o["scale"]))
    for i in range(len(pts)):
        for ob in range(off[i], off[i + 1]):
            Jp = oracle.ba_residual_jacobian(cams[cam[ob]], pts[i], f, *xy[ob].astype(float), mode=1)[2]
            Jsq[6 * len(cams) + 3 * i: 6 * len(cams) + 3 * i + 3] += (Jp ** 2).sum(0)
    scaled = Jsq[6 * len(cams):-1] * o["scale"][6 * len(cams):-1] ** 2
    assert (scaled < case["opts"]["min_lm_diagonal"]).sum() >= 5


_DENSE_OPTS = dict(max_num_iterations="max_num_iterations", function_tolerance="function_tolerance",
                   gradient_tolerance="gradient_tolerance", parameter_tolerance="parameter_tolerance",
                   initial_trust_region_radius="initial_radius", max_trust_region_radius="max_radius",
                   min_trust_region_radius="min_radius", min_relative_decrease="min_relative_decrease",
                   min_lm_diagonal="min_lm_diagonal", max_lm_diagonal="max_lm_diagonal",
                   max_num_consecutive_invalid_steps="max_consecutive_invalid")
# dense_lm does not test the cost for finiteness and always scales
_DENSE = [(k, n) for k, n in ALL if n != "eval_fail" and "no_scaling" not in n]


@pytest.mark.parametrize("kind,name", _DENSE, ids=[n for _, n in _DENSE])
def test_oracle_equals_dense_lm(oracle, kind, name):
    case = _case(kind, name)
    c, q, f, s, trace = _solve(oracle, case, jacobian_mode=0)
    d = dense_lm.solve(*case["args"], **{_DENSE_OPTS[k]: v for k, v in case["opts"].items()})
    assert ["CONVERGENCE", "NO_CONVERGENCE", "FAILURE"][s["termination_type"]] == d["termination"], (s, d["message"])
    assert (s["num_iterations"], s["num_successful_steps"]) == (d["iterations"], d["successful"])
    # the oracle (like the GPU solver) counts the invalid step that ends a FAILURE solve as unsuccessful; dense_lm stops
    # before counting it
    assert s["num_unsuccessful_steps"] == d["unsuccessful"] + (s["termination_type"] == bc.FAILURE)
    n = min(len(trace), len(d["costs"]))
    # the hard fixtures are ill-conditioned (far points, a 1 mm baseline): the two solvers' rounding separates the
    # trajectories by up to ~1e-8 relative, while every decision stays the same
    np.testing.assert_allclose(trace[:n, 0], d["costs"][:n], rtol=1e-7)
    # the radius follows rho = actual / model cost change, which those two fixtures' near-null directions make sensitive
    np.testing.assert_allclose(trace[:n, 1], d["radii"][:n], rtol=1e-3 if name in ("far_points", "short_baseline") else 1e-6)
    scale = max(1.0, np.abs(d["pts"]).max())
    if name in ("far_points", "short_baseline"):      # depths along a 1 mm baseline / at 1e5 m are barely determined
        np.testing.assert_allclose(c, d["cams"], rtol=1e-6, atol=1e-6)
    else:
        np.testing.assert_allclose(c, d["cams"], rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(q, d["pts"], rtol=1e-6, atol=1e-8 * scale)
    assert abs(f - d["focal"]) <= 1e-7 * max(1.0, abs(f))


@pytest.mark.parametrize("scaling", [0, 1])
@pytest.mark.parametrize("clamp", ["default", "binding"])
def test_reduced_system_with_non_default_options_is_the_dense_normal_equations(oracle, scaling, clamp):
    """The oracle's Schur-reduced system with jacobi_scaling 0/1 and clamp bounds that bind at both ends equals the Schur
    complement of the full damped normal equations built from dense_lm's complex-step Jacobian."""
    case = bc.wide()
    cams, pts, f, xy, cam, off = case["args"]
    bounds = bc.binding_bounds(oracle, case["args"], scaling) if clamp == "binding" else (1e-6, 1e32)
    obs_pt = np.repeat(np.arange(len(pts)), np.diff(off))
    J = dense_lm.dense_jacobian(np.asarray(cams, float), np.asarray(pts, float), f, xy.astype(float), cam.astype(np.int64), obs_pt)
    r = dense_lm.residuals(np.asarray(cams, float), np.asarray(pts, float), f, xy.astype(float), cam.astype(np.int64), obs_pt).reshape(-1)
    sc = 1.0 / (1.0 + np.sqrt((J * J).sum(0))) if scaling else np.ones(J.shape[1])
    Js = J * sc
    colsq = (Js * Js).sum(0)
    if clamp == "binding":
        assert (colsq < bounds[0]).sum() > 50 and (colsq > bounds[1]).sum() > 50
    for radius in (1e4, 3.7):
        H = Js.T @ Js + np.diag(np.clip(colsq, *bounds) / radius)
        b = Js.T @ r
        nc6, m = 6 * len(cams), len(cams) * 6 + 3 * len(pts)
        cf = np.r_[np.arange(nc6), [J.shape[1] - 1]]; pp = np.arange(nc6, m)
        Hpp_inv = np.linalg.inv(H[np.ix_(pp, pp)])
        S = H[np.ix_(cf, cf)] - H[np.ix_(cf, pp)] @ Hpp_inv @ H[np.ix_(pp, cf)]
        rhs = b[cf] - H[np.ix_(cf, pp)] @ Hpp_inv @ b[pp]
        o = oracle.ba_reduced_system(*case["args"], radius=radius, jacobi_scaling=scaling, min_diag=bounds[0], max_diag=bounds[1])
        assert o["ok"]
        np.testing.assert_allclose(o["S"], S, rtol=0, atol=1e-7 * np.abs(S).max())
        np.testing.assert_allclose(o["rhs"], rhs, rtol=0, atol=1e-7 * np.abs(rhs).max())
