"""GPU bundle adjustment (sfmb200_ba_*) against the oracle off the beaten path: every LM termination path, the state after
every iteration cap, non-default options at kernel level and in whole solves, the execution modes of the LM loop (chunks,
CUDA-graph replays, verbose, profile, L2 flush), a second run on the same handle, the time limit, and every track-length
dispatch bucket up to the 255 views per point the ABI accepts.  The fixtures (tests/ba_cases.py) are admissible: the oracle
takes the same decisions under its own rounding variations (tests/test_oracle_ba_lm_paths.py), so the GPU is held to them
exactly."""
import ctypes
import os
import re

import numpy as np
import pytest

import ba_cases as bc
from sfm_toy_library_b200 import capi, stages

pytestmark = pytest.mark.gpu
NTHR = max(1, min(32, os.cpu_count() or 1))
ILL = ("far_points", "short_baseline", "behind")     # depths along a 1 mm baseline / at 1e5 m / near a focal plane
NUM = re.compile(r"[-+]?\d+(?:\.\d*)?(?:[eE][-+]?\d+)?")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def gpu_opts(opts, **kw):
    return capi.ba_default_options(**{"max_solver_time_in_seconds": 0.0, **opts, **kw})


def oracle_solve(oracle, args, opts, **kw):
    o = oracle.ba_default_options(jacobian_mode=1, num_threads=NTHR, **{"max_solver_time_in_seconds": 0.0, **opts, **kw})
    return oracle.ba_solve(*args, o, want_trace=True)


def same_message(a, b):
    """Equal text once the numbers are taken out; the numbers to 1e-5 relative.  |cost_change| / cost of the function
    tolerance message is a difference of two costs that agree to ~1e-13 between the solvers: near 1e-9 that difference
    is only known to ~1e-13 absolute."""
    assert NUM.sub("#", a) == NUM.sub("#", b), (a, b)
    for x, y in zip(NUM.findall(a), NUM.findall(b)):
        assert abs(float(x) - float(y)) <= 1e-5 * abs(float(y)) + 1e-12, (a, b)


def cost_rtol(name):
    """1e-9; 1e-7 where the problem amplifies the solvers' rounding differences along the trajectory (every decision stays
    the same): near-null directions (ILL) and points close to the focal plane of a camera that sees them from behind.  The
    oracle and oracle/dense_lm.py differ by as much there (test_oracle_ba_lm_paths.py)."""
    return 1e-7 if name in ILL else 1e-9


def point_atol(name, args):
    """Per-point tolerance of the coordinates.  1e-8, except on the three ill-conditioned fixtures, where the measured
    spread between the oracle's own Jacobian modes sets it (with a 10x margin): 1e-7 everywhere on `behind`; on `far_points`
    1e-6 for the near points and 1e-4 of the depth for the points at 1e3..1e5; on `short_baseline` 1e-5 for the points of
    the circle and 1e-3 of the depth for the 2-view points of the 1 mm pair."""
    pts = np.asarray(args[1], float)
    dist = np.linalg.norm(pts, axis=1)
    if name == "far_points":
        return np.where(dist > 100, 1e-4 * dist, 1e-6)
    if name == "short_baseline":
        return np.where(np.diff(args[5]) == 2, 1e-3 * dist, 1e-5)
    return np.full(len(pts), 1e-7 if name == "behind" else 1e-8)


def expected_passes(s):
    """Residual+Jacobian passes (= linear solves) of a solve: one per LM iteration, plus the pass at the point where a test
    at the start of an iteration (gradient, radius, evaluation, or a cap of 0 iterations) stops it."""
    at_start = s["message"].startswith(("Gradient tolerance", "Minimum trust region radius", "Residual and Jacobian")) or \
        (s["num_iterations"] == 0 and s["message"].startswith("Maximum number of iterations"))
    return s["num_iterations"] + int(at_start)


def same_as_oracle(s, state, o, name="", params=True, args=None):
    cams, pts, f = state
    co, po, fo, so = o[:4]
    key = ("termination_type", "num_iterations", "num_successful_steps", "num_unsuccessful_steps")
    assert tuple(s[k] for k in key) == tuple(so[k] for k in key), (s, so)
    assert s["num_jacobian_passes"] == s["num_linear_solves"] == expected_passes(s), s
    same_message(s["message"], so["message"])
    if np.isfinite(so["final_cost"]):
        assert abs(s["initial_cost"] - so["initial_cost"]) <= 1e-12 * so["initial_cost"]
        assert abs(s["final_cost"] - so["final_cost"]) <= cost_rtol(name) * so["final_cost"], (s["final_cost"], so["final_cost"])
    if not params:
        return
    if name in ILL:
        np.testing.assert_allclose(cams, co, rtol=1e-6, atol=1e-6)
    else:
        np.testing.assert_allclose(cams, co, rtol=0, atol=1e-8)
    tol = point_atol(name, args) if args is not None else np.full(len(pts), 1e-8)
    bad = np.abs(np.asarray(pts) - po).max(1) > tol
    assert not bad.any(), (np.flatnonzero(bad)[:10], np.abs(np.asarray(pts) - po).max(1)[bad][:10])
    assert abs(f - fo) <= 1e-8 * max(1.0, abs(fo))


def run(ctx, args, options):
    prob = ctx.ba_problem(*args)
    try:
        return prob.run(options), prob.download()
    finally:
        prob.close()


# ---------------------------------------------------------------------------------------------------- termination paths
@pytest.mark.parametrize("name", list(bc.PATHS))
def test_termination_path_matches_oracle(ctx, oracle, name):
    case = bc.path_case(name)
    s, state = run(ctx, case["args"], gpu_opts(case["opts"]))
    o = oracle_solve(oracle, case["args"], case["opts"])
    assert s["termination_type"] == case["termination"] and s["message"].startswith(case["message"]), s
    same_as_oracle(s, state, o, name, args=case["args"])
    if case["termination"] == bc.FAILURE:                        # x never moved: the inputs, bit for bit
        cams, pts, f = state
        assert np.array_equal(cams, case["args"][0]) and np.array_equal(pts, case["args"][1]) and f == case["args"][2]
    if name == "eval_fail":
        assert s["num_iterations"] == 0 and not np.isfinite(s["initial_cost"])


def _adjust_bundle_inputs(args):
    """(cloud, poses, intrinsics, features) of stages.adjustBundle for a flattened problem (principal point 512, 384)."""
    cams, pts, f, xy, cam, off = args
    nc = len(cams)
    feats = [stages.Features(points=np.zeros((0, 2), np.float32)) for _ in range(nc)]
    by_view = [[] for _ in range(nc)]
    cloud = []
    for i in range(len(pts)):
        views = {}
        for o in range(off[i], off[i + 1]):
            v = int(cam[o]); views[v] = len(by_view[v]); by_view[v].append(xy[o] + np.float32([512, 384]))
        cloud.append(stages.Point3DInMap(pts[i].astype(np.float32), views))
    for v in range(nc):
        feats[v].points = np.array(by_view[v], np.float32).reshape(-1, 2)
    poses = []
    for c in cams:
        P = np.zeros((3, 4), np.float32); P[:, :3] = capi.angle_axis_to_rotmat(c[:3]); P[:, 3] = c[3:]; poses.append(P)
    K = np.array([[f, 0, 512], [0, f, 384], [0, 0, 1]], np.float32)
    return cloud, poses, stages.Intrinsics(K), feats


@pytest.mark.parametrize("name", ["point_fail_3", "eval_fail"])
def test_adjust_bundle_writes_nothing_back_on_failure(ctx, name):
    case = bc.path_case(name)
    cloud, poses, intr, feats = _adjust_bundle_inputs(case["args"])
    poses0 = [P.copy() for P in poses]; pts0 = np.array([q.p for q in cloud]); K0 = intr.K.copy()
    s = stages.adjustBundle(cloud, poses, intr, feats, ctx=ctx, options=gpu_opts(case["opts"]))
    assert s["termination_type"] == capi.FAILURE
    assert all(np.array_equal(a, b) for a, b in zip(poses, poses0)) and np.array_equal(np.array([q.p for q in cloud]), pts0)
    assert np.array_equal(intr.K, K0)


def test_adjust_bundle_leaves_out_the_camera_nobody_observes(ctx):
    """The chol-fail path needs a camera without observations in the problem.  adjustBundle never builds one: like Ceres,
    which only sees parameter blocks that carry a residual, it flattens the observed views only.  On the chol-fail inputs it
    therefore converges, and the unobserved camera's pose only goes through the float angle-axis round trip the reference
    applies to every pose after CONVERGENCE (DESIGN.md section 1): its translation is unchanged."""
    case = bc.path_case("chol_fail_3")
    assert 6 not in case["args"][4]
    cloud, poses, intr, feats = _adjust_bundle_inputs(case["args"])
    pose6 = poses[6].copy()
    s = stages.adjustBundle(cloud, poses, intr, feats, ctx=ctx, options=gpu_opts(case["opts"]))
    assert s["termination_type"] == capi.CONVERGENCE
    assert np.array_equal(poses[6][:, 3], pose6[:, 3]) and np.abs(poses[6] - pose6).max() < 1e-6


# ------------------------------------------------------------------------------------------------ per-iteration trajectory
TRAJ = ["wide", "far_points", "short_baseline", "outliers", "behind", "ragged"]


@pytest.mark.parametrize("name", TRAJ)
def test_state_after_every_iteration_cap(ctx, oracle, name):
    """max_num_iterations = k for every k up to the oracle's count, caps on rejected steps included: summary and state equal
    the oracle's with the same cap, final_cost is the oracle trace's cost after iteration k, and the accepted steps so far
    are the trace's."""
    case = bc.FIXTURES[name]()
    full = oracle_solve(oracle, case["args"], case["opts"])
    trace = full[4]
    n = full[3]["num_iterations"]
    prob = ctx.ba_problem(*case["args"])
    try:
        for k in range(n + 1):
            prob.reset()
            s = prob.run(gpu_opts(case["opts"], max_num_iterations=k))
            state = prob.download()
            same_as_oracle(s, state, oracle_solve(oracle, case["args"], case["opts"], max_num_iterations=k), name, args=case["args"])
            assert abs(s["final_cost"] - trace[k, 0]) <= cost_rtol(name) * trace[k, 0], (k, s["final_cost"], trace[k, 0])
            assert s["num_successful_steps"] == int((trace[1:k + 1, 2] == 1).sum()), k
    finally:
        prob.close()
    assert (trace[1:, 2] == 0).any() or name in ("far_points", "outliers", "behind", "ragged")


def test_verbose_lines_follow_the_oracle_trace(ctx, oracle, capfd):
    """verbose = 1 prints one line per LM iteration: its cost and radius are the oracle trace's after that iteration, its
    |g|max that of the point the iteration started from (the gradient at an accepted point is evaluated by the next pass)."""
    case = bc.FIXTURES["wide"]()
    trace = oracle_solve(oracle, case["args"], case["opts"])[4]
    libc = ctypes.CDLL(None)
    libc.fflush(None); capfd.readouterr()
    s, _ = run(ctx, case["args"], gpu_opts(case["opts"], verbose=1))
    libc.fflush(None)
    lines = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("iter ")]
    pat = re.compile(r"iter\s+(\d+) cost (\S+) \|g\|max (\S+) radius (\S+) rho (\S+) (ok|rejected|stop)$")
    assert len(lines) >= s["num_iterations"]
    prev = -1
    for ln in lines:
        m = pat.match(ln)
        assert m, ln
        i, cost, gmax, radius = int(m.group(1)), float(m.group(2)), float(m.group(3)), float(m.group(4))
        assert abs(cost - trace[i, 0]) <= 1e-9 * trace[i, 0], (ln, trace[i])
        assert abs(radius - trace[i, 1]) <= 1e-3 * trace[i, 1], (ln, trace[i])
        g_ref = trace[i, 3] if (m.group(6) == "stop" and i == prev) else trace[i - 1, 3]
        assert abs(gmax - g_ref) <= 1e-3 * g_ref, (ln, g_ref)
        assert (m.group(6) == "ok") == (m.group(6) != "stop" and trace[i, 2] == 1), (ln, trace[i])
        prev = i
    assert prev == s["num_iterations"]


# ---------------------------------------------------------------------------------------- non-default options, kernel level
@pytest.mark.parametrize("scaling", [0, 1])
@pytest.mark.parametrize("clamp", ["default", "binding"])
def test_reduced_system_with_non_default_options(ctx, oracle, scaling, clamp):
    """jacobi_scaling 0 / 1 and an LM diagonal clamp that binds at both ends: the point kernel's, the assembly's and (through
    whole solves) the camera update's clamps all take the options."""
    case = bc.FIXTURES["wide"]()
    lo, hi = bc.binding_bounds(oracle, case["args"], scaling) if clamp == "binding" else (1e-6, 1e32)
    opts = dict(jacobi_scaling=scaling, min_lm_diagonal=lo, max_lm_diagonal=hi)
    prob = ctx.ba_problem(*case["args"])
    try:
        for radius in (1e4, 3.7):
            g = prob.reduced_system(radius, gpu_opts(opts))
            o = oracle.ba_reduced_system(*case["args"], radius=radius, jacobi_scaling=scaling, min_diag=lo, max_diag=hi)
            n = 6 * len(case["args"][0])
            assert abs(g["cost"] - o["cost"]) < 1e-12 * o["cost"]
            np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
            np.testing.assert_allclose(g["rhs"], o["rhs"], rtol=0, atol=1e-10 * np.abs(o["rhs"]).max())
            gcf = np.concatenate([o["grad"][:n], o["grad"][-1:]])
            np.testing.assert_allclose(g["grad_cf"], gcf, rtol=1e-9, atol=1e-9 * np.abs(gcf).max())
    finally:
        prob.close()


# ------------------------------------------------------------------------------------------------------- execution modes
def _large():
    from sfm_toy_library_b200 import synth
    p = synth.make_ba_problem(n_cams=20, n_pts=12600, obs_per_pt=8, seed=1)     # 100,800 observations: no graph, chunks of 4
    return dict(args=bc.args_of(p), opts={})


MODES = [("chunk1", {"SFMB200_BA_CHUNK": "1"}, {}), ("chunk3", {"SFMB200_BA_CHUNK": "3"}, {}),
         ("chunk16", {"SFMB200_BA_CHUNK": "16"}, {}), ("nograph", {"SFMB200_BA_GRAPH": "0"}, {}),
         ("verbose", {}, dict(verbose=1)), ("profile", {}, dict(profile=1)), ("flush", {}, dict(l2_flush_mb=64))]
VOLATILE = ("total_time_s", "schur_ms_total", "schur_launches", "pair_ms_total", "pair_launches", "camera_ms_total",
            "solve_ms_total", "flush_ms_total", "kernel_launches")


@pytest.mark.parametrize("size", ["small", "large"])
def test_execution_modes_give_the_same_bits(ctx, oracle, monkeypatch, size):
    """Chunks of 1, 3 and 16 iterations, no CUDA graph, verbose, profile and L2 flushing issue the same LM iterations: same
    summary, pass and solve counts included, and the same parameter bits.  The small problem (26 iterations) ends inside a
    graph replay, the large one (3 iterations) inside its first chunk: the iterations enqueued after the end do not count."""
    case = bc.FIXTURES["wide"]() if size == "small" else _large()
    ref = run(ctx, case["args"], gpu_opts(case["opts"]))
    assert ref[0]["num_iterations"] % 4 != 0
    same_as_oracle(*ref, oracle_solve(oracle, case["args"], case["opts"]), params=size == "small")
    assert ref[0]["num_jacobian_passes"] == ref[0]["num_iterations"]
    for mode, env, kw in MODES:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            s, state = run(ctx, case["args"], gpu_opts(case["opts"], **kw))
        for k in ref[0]:
            if k not in VOLATILE:
                assert s[k] == ref[0][k], (mode, k, s[k], ref[0][k])
        assert all(np.array_equal(a, b) for a, b in zip(state[:2], ref[1][:2])) and state[2] == ref[1][2], mode


def test_second_run_without_reset_continues_from_the_first(ctx, oracle):
    case = bc.FIXTURES["wide"]()
    prob = ctx.ba_problem(*case["args"])
    try:
        prob.run(gpu_opts(case["opts"], max_num_iterations=5))
        mid = prob.download()
        s = prob.run(gpu_opts(case["opts"]))
        state = prob.download()
    finally:
        prob.close()
    a = case["args"]
    same_as_oracle(s, state, oracle_solve(oracle, (mid[0], mid[1], mid[2]) + tuple(a[3:]), case["opts"]), "wide")


def test_time_limit_stops_between_chunks(ctx, oracle):
    case = bc.FIXTURES["wide"]()
    s, state = run(ctx, case["args"], gpu_opts(case["opts"], max_solver_time_in_seconds=1e-9))
    assert s["termination_type"] == capi.NO_CONVERGENCE and s["message"] == "Maximum solver time reached.", s
    assert 0 < s["num_iterations"] < 26 and s["num_jacobian_passes"] == s["num_linear_solves"] == s["num_iterations"]
    s2, state2 = run(ctx, case["args"], gpu_opts(case["opts"], max_num_iterations=s["num_iterations"]))
    assert all(np.array_equal(a, b) for a, b in zip(state[:2], state2[:2])) and state[2] == state2[2]
    assert s2["final_cost"] == s["final_cost"]
    c = oracle.ba_cost(*state, *case["args"][3:])
    assert abs(c - s["final_cost"]) <= 1e-12 * c


# --------------------------------------------------------------------------------------------------- track-length buckets
@pytest.mark.parametrize("maxk", [4, 5, 8, 9, 16, 17, 32, 33, 60, 120, 244, 245, 255])
def test_track_length_buckets(ctx, oracle, maxk):
    """G = 4 / 8 / 16 / 32 lanes per point, staged (maxk <= G) and unstaged, up to the 255 views the ABI accepts:
    reduced system and a three-iteration solve against the oracle."""
    case = bc.track_lengths(maxk)
    assert np.diff(case["args"][5]).max() == maxk
    assert capi.ba_validate(len(case["args"][0]), case["args"][4], case["args"][5])[0] == 0
    prob = ctx.ba_problem(*case["args"])
    try:
        g = prob.reduced_system(1e4)
        o = oracle.ba_reduced_system(*case["args"], radius=1e4)
        np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
        np.testing.assert_allclose(g["rhs"], o["rhs"], rtol=0, atol=1e-10 * np.abs(o["rhs"]).max())
        s = prob.run(gpu_opts({}, max_num_iterations=3))
        state = prob.download()
    finally:
        prob.close()
    same_as_oracle(s, state, oracle_solve(oracle, case["args"], {}, max_num_iterations=3))


def test_ragged_tracks_with_empty_and_single_view_points(ctx, oracle):
    case = bc.FIXTURES["ragged"]()
    lens = np.diff(case["args"][5])
    assert (lens == 0).any() and (lens == 1).any() and lens.max() == 60
    prob = ctx.ba_problem(*case["args"])
    try:
        for radius in (1e4, 3.7):
            g = prob.reduced_system(radius)
            o = oracle.ba_reduced_system(*case["args"], radius=radius)
            np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
            np.testing.assert_allclose(g["rhs"], o["rhs"], rtol=0, atol=1e-10 * np.abs(o["rhs"]).max())
    finally:
        prob.close()


def _error_code(e):
    return int(re.search(r"error (-?\d+)", str(e)).group(1))


def test_256_views_refused_alike_by_validate_and_create(ctx):
    case = bc.track_lengths(255, n_cams=260)
    cam, off = case["args"][4], case["args"][5]
    # one more view for the first point
    extra = np.setdiff1d(np.arange(260), cam[off[0]:off[1]])[0]
    cam = np.r_[np.sort(np.r_[cam[off[0]:off[1]], extra]), cam[off[1]:]].astype(np.int32)
    xy = np.r_[case["args"][3][:1], case["args"][3]].astype(np.float32)
    off = np.r_[0, off[1:] + 1].astype(np.int32)
    rc, msg = capi.ba_validate(260, cam, off)
    assert rc != 0 and msg == "a point is observed by 256 views; at most 255 supported"
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.ba_problem(case["args"][0], case["args"][1], case["args"][2], xy, cam, off)
    assert _error_code(e.value) == rc and str(e.value).endswith(msg)


@pytest.mark.parametrize("maxk", [244, 245, 255])
def test_red_schur_mode_view_limit(ctx, oracle, monkeypatch, maxk):
    """What validate accepts, create accepts in the default gather mode (above); the atomics ("red") mode keeps a point's
    Schur terms in shared memory, takes up to 244 views and refuses more with the message the header documents."""
    case = bc.track_lengths(maxk)
    monkeypatch.setenv("SFMB200_BA_SCHUR", "red")
    if maxk <= 244:
        prob = ctx.ba_problem(*case["args"])
        try:
            g = prob.reduced_system(1e4)
        finally:
            prob.close()
        o = oracle.ba_reduced_system(*case["args"], radius=1e4)
        np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
        return
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.ba_problem(*case["args"])
    assert str(e.value).endswith('observations per point (%d) exceed the shared-memory budget of the atomics ("red") Schur mode' % maxk)
    assert capi.ba_validate(len(case["args"][0]), case["args"][4], case["args"][5])[0] == 0


def test_view_limits_are_documented_as_enforced():
    """The header and DESIGN.md state the limits the two calls enforce: 255 views for validate and gather-mode create,
    244 in red mode, with create's refusal message; the red-mode bound is the shared-memory formula at 200 KB."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = " ".join(open(os.path.join(root, "include", "sfmb200.h")).read().split()).replace(" * ", " ")
    design = " ".join(open(os.path.join(root, "DESIGN.md")).read().split())
    msg = 'exceed the shared-memory budget of the atomics ("red") Schur mode'
    assert "at most 255 views per point" in hdr and "at most 244 views per point" in hdr and msg in hdr
    assert "accepts at most 255" in design and "at most 244 views per point" in design and msg in design
    smem = lambda k: k * k + 591 * k + 16                      # point_smem_bytes(32, k) (ba.cu), documented in DESIGN.md
    assert "maxk² + 591·maxk + 16" in design and smem(244) <= 200 * 1024 < smem(245)
