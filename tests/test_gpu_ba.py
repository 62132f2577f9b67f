"""GPU parity: sfmb200_ba_* (CUDA, through the C ABI) vs the oracle restatement of adjustBundle / Ceres LM + DENSE_SCHUR
(SfMBundleAdjustmentUtils.cpp:58-222).  north_star tolerance: reprojection error within 1e-4 px."""
import numpy as np
import pytest

from sfm_toy_library_b200 import capi, stages, synth

pytestmark = pytest.mark.gpu
PX_TOL = 1e-4


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _args(p):
    return p["cams"], p["pts"], p["focal"], p["obs_xy"], p["obs_cam"], p["pt_off"]


def _residuals(oracle, cams, pts, f, p):
    r = np.empty((p["nobs"], 2))
    for o in range(p["nobs"]):
        r[o] = oracle.ba_residual_jacobian(cams[p["obs_cam"][o]], pts[p["obs_pt"][o]], f, *p["obs_xy"][o].astype(float), mode=1)[0]
    return r


@pytest.mark.parametrize("nc,npts,k,seed", [(4, 30, 3, 5), (6, 150, 4, 11), (20, 2000, 8, 0), (7, 400, 2, 3), (40, 500, 20, 4)])
def test_reduced_system_matches_oracle(ctx, oracle, nc, npts, k, seed):
    """Kernel-level: S, rhs, gradient, cost of one residual+Jacobian+Schur pass (K3a + K3b + assemble)."""
    p = synth.make_ba_problem(n_cams=nc, n_pts=npts, obs_per_pt=k, seed=seed)
    prob = ctx.ba_problem(*_args(p))
    for radius in (1e4, 3.7):
        g = prob.reduced_system(radius)
        o = oracle.ba_reduced_system(*_args(p), radius=radius)
        n = 6 * nc
        assert abs(g["cost"] - o["cost"]) < 1e-12 * o["cost"]
        scale = np.abs(o["S"]).max()
        np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * scale)
        np.testing.assert_allclose(g["rhs"], o["rhs"], rtol=0, atol=1e-10 * np.abs(o["rhs"]).max())
        gcf = np.concatenate([o["grad"][:n], o["grad"][-1:]])
        np.testing.assert_allclose(g["grad_cf"], gcf, rtol=1e-9, atol=1e-9 * np.abs(gcf).max())
    prob.close()


@pytest.mark.parametrize("nc,npts,k,seed", [(6, 150, 4, 11), (20, 2000, 8, 0), (12, 800, 3, 7)])
def test_solve_matches_oracle_trajectory(ctx, oracle, nc, npts, k, seed):
    p = synth.make_ba_problem(n_cams=nc, n_pts=npts, obs_per_pt=k, seed=seed)
    cams, pts, f, s = ctx.ba_solve(*_args(p))
    co, po, fo, so = oracle.ba_solve(*_args(p), oracle.ba_default_options(jacobian_mode=0))
    assert s["termination_type"] == so["termination_type"] == capi.CONVERGENCE, (s, so)
    assert s["num_iterations"] == so["num_iterations"] and s["num_successful_steps"] == so["num_successful_steps"], (s, so)
    assert abs(s["initial_cost"] - so["initial_cost"]) < 1e-12 * so["initial_cost"]
    assert abs(s["final_cost"] - so["final_cost"]) < 1e-9 * so["final_cost"]
    # reprojection residual of every observation within 1e-4 px of the reference path's
    assert np.abs(_residuals(oracle, cams, pts, f, p) - _residuals(oracle, co, po, fo, p)).max() < PX_TOL
    assert abs(f - fo) < 1e-6 * fo


def test_golden_scipy_optimum(ctx, golden):
    g = golden("ba_scipy.npz")
    o = capi.ba_default_options(max_solver_time_in_seconds=0.0, function_tolerance=1e-12, parameter_tolerance=1e-12, max_num_iterations=200)
    cams, pts, f, s = ctx.ba_solve(g["cams"], g["pts"], float(g["focal"]), g["obs_xy"], g["obs_cam"], g["pt_off"], o)
    assert s["termination_type"] == capi.CONVERGENCE
    assert abs(s["initial_cost"] - float(g["cost0"])) < 1e-9 * float(g["cost0"])
    assert abs(s["final_cost"] - float(g["cost_opt"])) < 2e-3 * float(g["cost_opt"])


def test_problem_handle_reset_and_rerun_is_reproducible(ctx):
    p = synth.make_ba_problem(n_cams=10, n_pts=1000, obs_per_pt=5, seed=9)
    prob = ctx.ba_problem(*_args(p))
    s1 = prob.run(); c1, p1, f1 = prob.download()
    prob.reset()
    s2 = prob.run(); c2, p2, f2 = prob.download()
    assert s1["num_iterations"] == s2["num_iterations"] and s1["termination_type"] == capi.CONVERGENCE
    np.testing.assert_allclose(c1, c2, rtol=0, atol=1e-9); np.testing.assert_allclose(p1, p2, rtol=0, atol=1e-9)
    assert s1["kernel_launches"] > 0 and s1["num_jacobian_passes"] >= s1["num_iterations"]
    prob.close()


def test_iteration_cap_gives_no_convergence_and_adjustbundle_discards(ctx):
    """adjustBundle writes nothing back unless Ceres reports CONVERGENCE (SfMBundleAdjustmentUtils.cpp:182-185)."""
    p = synth.make_ba_problem(n_cams=5, n_pts=200, obs_per_pt=3, seed=21)
    K = np.array([[p["focal"], 0, 512], [0, p["focal"], 384], [0, 0, 1]], np.float32)
    feats = [stages.Features(points=np.zeros((0, 2), np.float32)) for _ in range(5)]
    pts_by_view = [[] for _ in range(5)]
    cloud = []
    for i in range(p["np"]):
        views = {}
        for o in range(p["pt_off"][i], p["pt_off"][i + 1]):
            v = int(p["obs_cam"][o]); views[v] = len(pts_by_view[v]); pts_by_view[v].append(p["obs_xy"][o] + np.float32([512, 384]))
        cloud.append(stages.Point3DInMap(p["pts"][i].astype(np.float32), views))
    for v in range(5):
        feats[v].points = np.array(pts_by_view[v], np.float32).reshape(-1, 2)
    poses = []
    for c in p["cams"]:
        P = np.zeros((3, 4), np.float32); P[:, :3] = synth.angle_axis_to_rotmat(c[:3]); P[:, 3] = c[3:]; poses.append(P)
    poses0 = [P.copy() for P in poses]; pts0 = np.array([q.p for q in cloud])
    intr = stages.Intrinsics(K.copy())
    s = stages.adjustBundle(cloud, poses, intr, feats, ctx=ctx, options=capi.ba_default_options(max_num_iterations=1))
    assert s["termination_type"] == capi.NO_CONVERGENCE
    assert all(np.array_equal(a, b) for a, b in zip(poses, poses0)) and np.array_equal(np.array([q.p for q in cloud]), pts0)
    assert intr.K[0, 0] == K[0, 0]
    s = stages.adjustBundle(cloud, poses, intr, feats, ctx=ctx)
    assert s["termination_type"] == capi.CONVERGENCE and s["final_cost"] < 1e-3 * s["initial_cost"]
    assert not np.array_equal(np.array([q.p for q in cloud]), pts0) and intr.K[0, 0] == intr.K[1, 1] != K[0, 0]
    assert abs(float(intr.K[0, 0]) - p["focal_true"]) < 10


def test_degenerate_inputs(ctx):
    p = synth.make_ba_problem(n_cams=3, n_pts=10, obs_per_pt=2, seed=1)
    with pytest.raises(capi.SfmB200Error):                                   # cameras must ascend within a point
        ctx.ba_solve(p["cams"], p["pts"], p["focal"], p["obs_xy"], p["obs_cam"][::-1].copy(), p["pt_off"])
    # perfect data: zero cost -> gradient tolerance at iteration 0
    q = synth.make_ba_problem(n_cams=4, n_pts=50, obs_per_pt=3, seed=2, noise_px=0.0, perturb=False)
    cams, pts, f, s = ctx.ba_solve(*_args(q))
    assert s["termination_type"] == capi.CONVERGENCE and s["final_cost"] < 1e-3   # float32 observations leave ~1e-5 px
    # a camera nobody observes stays put
    r = synth.make_ba_problem(n_cams=6, n_pts=300, obs_per_pt=3, seed=3)
    keep = r["obs_cam"] != 5
    ok_pts = np.array([keep[r["pt_off"][i]:r["pt_off"][i + 1]].all() for i in range(r["np"])])
    sel = np.repeat(ok_pts, 3)
    off = np.arange(ok_pts.sum() + 1, dtype=np.int32) * 3
    cams, pts, f, s = ctx.ba_solve(r["cams"], r["pts"][ok_pts], r["focal"], r["obs_xy"][sel], r["obs_cam"][sel], off)
    assert s["termination_type"] == capi.CONVERGENCE
    np.testing.assert_array_equal(cams[5], r["cams"][5])


def test_config2_full_size(ctx, oracle):
    """BASELINE.json configs[1]: 20 cams / 10k points / 80k observations, against the oracle (seconds on the CPU)."""
    p = synth.make_ba_problem(**synth.BA_CONFIGS["cfg2"])
    cams, pts, f, s = ctx.ba_solve(*_args(p))
    co, po, fo, so = oracle.ba_solve(*_args(p), oracle.ba_default_options(jacobian_mode=1))
    assert s["termination_type"] == so["termination_type"] == capi.CONVERGENCE
    assert s["num_iterations"] == so["num_iterations"]
    assert abs(s["final_cost"] - so["final_cost"]) < 1e-9 * so["final_cost"]
    rms = np.sqrt(2 * s["final_cost"] / p["nobs"])
    assert 0.55 < rms < 0.75
    np.testing.assert_allclose(pts, po, rtol=0, atol=1e-7); np.testing.assert_allclose(cams, co, rtol=0, atol=1e-7)


def test_config3_properties_full_size(ctx, oracle):
    """BASELINE.json configs[2]: 100 cams / 200k points / 1.6M observations.  Size-independent checks: cost decreases
    monotonically to the noise floor, the oracle's cost function agrees at the returned point, the optimum is
    stationary (re-running from it converges immediately)."""
    p = synth.make_ba_problem(**synth.BA_CONFIGS["cfg3"])
    prob = ctx.ba_problem(*_args(p))
    s = prob.run(capi.ba_default_options(max_solver_time_in_seconds=0.0))
    cams, pts, f = prob.download()
    assert s["termination_type"] == capi.CONVERGENCE and s["num_iterations"] <= 20
    rms = np.sqrt(2 * s["final_cost"] / p["nobs"])
    assert 0.6 < rms < 0.75
    c = oracle.ba_cost(cams, pts, f, p["obs_xy"], p["obs_cam"], p["pt_off"], nthreads=4)
    assert abs(c - s["final_cost"]) < 1e-10 * c
    s2 = ctx.ba_solve(cams, pts, f, p["obs_xy"], p["obs_cam"], p["pt_off"])[3]
    assert s2["termination_type"] == capi.CONVERGENCE and s2["num_iterations"] <= 2
    prob.close()


def test_red_and_gather_schur_modes_agree(ctx, oracle, monkeypatch):
    """The two implementations of the off-diagonal Schur blocks (atomics-free per-camera-pair gather, default, and the
    per-point RED sweep) give the same reduced system and the same solve."""
    p = synth.make_ba_problem(n_cams=12, n_pts=1500, obs_per_pt=5, seed=13)
    out = {}
    for mode in ("gather", "red"):
        monkeypatch.setenv("SFMB200_BA_SCHUR", mode)
        prob = ctx.ba_problem(*_args(p))
        out[mode] = (prob.reduced_system(1e4), prob.run(), prob.download())
        prob.close()
    o = oracle.ba_reduced_system(*_args(p), radius=1e4)
    for mode in ("gather", "red"):
        np.testing.assert_allclose(out[mode][0]["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
    assert out["gather"][1]["num_iterations"] == out["red"][1]["num_iterations"]
    assert abs(out["gather"][1]["final_cost"] - out["red"][1]["final_cost"]) < 1e-10 * out["red"][1]["final_cost"]
    np.testing.assert_allclose(out["gather"][2][1], out["red"][2][1], rtol=0, atol=1e-8)


@pytest.mark.parametrize("n_cams,n_pts,k,iters", [(5, 400, 5, 8), (40, 3000, 6, 8), (100, 6000, 6, 8), (180, 5000, 6, 8), (480, 3000, 4, 3)])
def test_dense_solve_matches_oracle_trajectory(ctx, oracle, n_cams, n_pts, k, iters):
    """The dense solve (dataflow tile Cholesky + back substitution) inside whole LM iterations, against the oracle's trajectory.
    1 / 8 / 19 / 34 tile rows; 180 cameras have more tiles (595) than co-resident CTAs, so CTAs own several tiles.  Up to
    469 cameras (n = 6 cams + 1 <= 2816) the back substitution runs on a CTA cluster; 480 cameras (n = 2881) are past the
    cluster kernel's shared-memory limit and take the single-CTA back substitution."""
    import os
    p = synth.make_ba_problem(n_cams=n_cams, n_pts=n_pts, obs_per_pt=k, seed=21)
    opts = dict(max_num_iterations=iters, max_solver_time_in_seconds=0.0)
    prob = ctx.ba_problem(*_args(p))
    a = (prob.run(capi.ba_default_options(**opts)), prob.download())
    prob.close()
    nthr = max(1, min(32, (os.cpu_count() or 1)))
    co, po, fo, so = oracle.ba_solve(*_args(p), oracle.ba_default_options(jacobian_mode=1, num_threads=nthr, **opts))
    assert (a[0]["num_successful_steps"], a[0]["num_unsuccessful_steps"]) == (so["num_successful_steps"], so["num_unsuccessful_steps"]), (a[0], so)
    _same_trajectory(a, (so, (co, po, fo)))


def _same_trajectory(a, b):
    assert a[0]["termination_type"] == b[0]["termination_type"] and a[0]["num_iterations"] == b[0]["num_iterations"]
    assert a[0]["final_cost"] < 0.1 * a[0]["initial_cost"]
    assert abs(a[0]["final_cost"] - b[0]["final_cost"]) < 1e-9 * b[0]["final_cost"]
    np.testing.assert_allclose(a[1][0], b[1][0], rtol=0, atol=1e-8)
    np.testing.assert_allclose(a[1][1], b[1][1], rtol=0, atol=1e-8)


def test_backsubstitution_from_stored_blocks_matches_jacobian_path(ctx, monkeypatch):
    """Default back-substitution (stored Z blocks, model cost change as 1/2 y.(g + D^2 y)) against the kernel that
    re-evaluates the Jacobians and forms Ceres' -m.(r + m/2): same LM trajectory, accepted and rejected steps alike."""
    p = synth.make_ba_problem(n_cams=30, n_pts=4000, obs_per_pt=7, seed=33)
    out = {}
    for mode in ("stored", "jacobian"):
        monkeypatch.setenv("SFMB200_BA_BACKSUB", mode)
        prob = ctx.ba_problem(*_args(p))
        o = capi.ba_default_options(); o.max_num_iterations = 12; o.initial_trust_region_radius = 1e2    # small radius: some steps get rejected
        out[mode] = (prob.run(o), prob.download())
        prob.close()
    a, b = out["stored"], out["jacobian"]
    assert a[0]["num_successful_steps"] == b[0]["num_successful_steps"] and a[0]["num_unsuccessful_steps"] == b[0]["num_unsuccessful_steps"]
    _same_trajectory(a, b)


def test_many_observations_per_point_and_ragged_tracks(ctx, oracle):
    """Track lengths 2..40 in one problem (G = 32 groups, multi-chunk points, long pair lists)."""
    rs = np.random.RandomState(5)
    base = synth.make_ba_problem(n_cams=40, n_pts=300, obs_per_pt=40, seed=6)
    keep = np.zeros(base["nobs"], bool); off = [0]
    for i in range(base["np"]):
        k = int(rs.randint(2, 41))
        sel = np.sort(rs.choice(40, k, replace=False)) + base["pt_off"][i]
        keep[sel] = True; off.append(off[-1] + k)
    args = (base["cams"], base["pts"], base["focal"], base["obs_xy"][keep], base["obs_cam"][keep], np.asarray(off, np.int32))
    prob = ctx.ba_problem(*args)
    g = prob.reduced_system(1e4); o = oracle.ba_reduced_system(*args, radius=1e4)
    np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
    np.testing.assert_allclose(g["rhs"], o["rhs"], rtol=0, atol=1e-10 * np.abs(o["rhs"]).max())
    s = prob.run(); so = oracle.ba_solve(*args, oracle.ba_default_options(jacobian_mode=1))[3]
    assert s["termination_type"] == so["termination_type"] and s["num_iterations"] == so["num_iterations"]
    assert abs(s["final_cost"] - so["final_cost"]) < 1e-9 * so["final_cost"]
    prob.close()


def test_config3_trajectory_vs_oracle_full_size(ctx, oracle):
    """The headline configuration (BASELINE configs[2]: 100 cameras / 200 k points / 1.6 M observations) against the oracle's
    whole LM trajectory (all host threads, ~0.1 s per iteration): same termination, same number of iterations, accepted
    and rejected steps, final cost to 1e-9, every camera to 1e-7, reprojection residuals within north_star's 1e-4 px."""
    import os
    p = synth.make_ba_problem(**synth.BA_CONFIGS["cfg3"])
    opts = dict(max_solver_time_in_seconds=0.0)                       # the 10 s cap (:176) is a property of the host clock, not of the algorithm
    prob = ctx.ba_problem(*_args(p))
    s = prob.run(capi.ba_default_options(**opts))
    cams, pts, f = prob.download()
    prob.close()
    nthr = max(1, min(32, (os.cpu_count() or 1)))
    co, po, fo, so, trace = oracle.ba_solve(*_args(p), oracle.ba_default_options(jacobian_mode=1, num_threads=nthr, **opts), want_trace=True)
    assert s["termination_type"] == so["termination_type"] == capi.CONVERGENCE, (s, so)
    assert (s["num_iterations"], s["num_successful_steps"], s["num_unsuccessful_steps"]) == \
           (so["num_iterations"], so["num_successful_steps"], so["num_unsuccessful_steps"]), (s, so)
    assert abs(s["initial_cost"] - so["initial_cost"]) < 1e-12 * so["initial_cost"]
    assert abs(s["final_cost"] - so["final_cost"]) < 1e-9 * so["final_cost"]
    np.testing.assert_allclose(cams, co, rtol=0, atol=1e-7)
    assert abs(f - fo) < 1e-7 * fo
    np.testing.assert_allclose(pts, po, rtol=0, atol=1e-7)
    # reprojection residuals, vectorised (1.6 M observations)
    def res(c, q, ff):
        R = np.stack([capi.angle_axis_to_rotmat(x[:3]) for x in c])
        P = np.einsum("oij,oj->oi", R[p["obs_cam"]], q[p["obs_pt"]]) + c[p["obs_cam"], 3:]
        return ff * P[:, :2] / P[:, 2:3] - p["obs_xy"]
    assert np.abs(res(cams, pts, f) - res(co, po, fo)).max() < PX_TOL


def test_config2_reaches_the_independent_scipy_optimum(ctx, golden):
    """cfg 2 at full size against tests/golden/ba_scipy_cfg2.npz (scipy TRF, complex-step sparse Jacobian of an independent
    numpy model): cost within 1e-9 with tight tolerances, within 1e-6 with Ceres' defaults; focal (gauge invariant) to 1e-5."""
    g = golden("ba_scipy_cfg2.npz")
    p = synth.make_ba_problem(seed=0, **synth.BA_CONFIGS["cfg2"])
    o = capi.ba_default_options(max_solver_time_in_seconds=0.0, function_tolerance=1e-14, parameter_tolerance=1e-14, max_num_iterations=60)
    cams, pts, f, s = ctx.ba_solve(*_args(p), o)
    assert abs(s["initial_cost"] - float(g["cost0"])) < 1e-10 * float(g["cost0"])
    assert abs(s["final_cost"] - float(g["cost_opt"])) < 1e-9 * float(g["cost_opt"]), (s["final_cost"], float(g["cost_opt"]))
    assert abs(f - float(g["focal"])) < 1e-5 * f
    s = ctx.ba_solve(*_args(p), capi.ba_default_options(max_solver_time_in_seconds=0.0))[3]
    assert s["termination_type"] == capi.CONVERGENCE and 0 <= s["final_cost"] - float(g["cost_opt"]) < 1e-6 * float(g["cost_opt"])


@pytest.mark.parametrize("nc,npts,k,seed", [(4, 60, 3, 5), (6, 150, 4, 11), (10, 300, 5, 2)])
def test_trajectory_equals_independent_dense_lm(ctx, nc, npts, k, seed):
    """GPU vs oracle/dense_lm.py (explicit dense Jacobian by complex-step differentiation, full normal equations, Ceres'
    update rules written from the Ceres documentation): same accept/reject sequence, termination and final state."""
    from oracle import dense_lm
    p = synth.make_ba_problem(n_cams=nc, n_pts=npts, obs_per_pt=k, seed=seed)
    cams, pts, f, s = ctx.ba_solve(*_args(p), capi.ba_default_options(max_solver_time_in_seconds=0.0))
    d = dense_lm.solve(*_args(p))
    assert ["CONVERGENCE", "NO_CONVERGENCE", "FAILURE"][s["termination_type"]] == d["termination"]
    assert (s["num_iterations"], s["num_successful_steps"], s["num_unsuccessful_steps"]) == (d["iterations"], d["successful"], d["unsuccessful"])
    assert abs(s["final_cost"] - d["final_cost"]) < 1e-9 * d["final_cost"]
    np.testing.assert_allclose(cams, d["cams"], rtol=1e-7, atol=1e-9); np.testing.assert_allclose(pts, d["pts"], rtol=1e-7, atol=1e-9)


def test_two_runs_are_bitwise_identical(ctx):
    """Deterministic summation order everywhere (camera-pair entry lists sorted by point once per problem, fixed-shape
    reductions): re-running a problem, and re-creating it, reproduces every parameter bit for bit (SURVEY.md 7)."""
    p = synth.make_ba_problem(n_cams=24, n_pts=5000, obs_per_pt=6, seed=17)
    outs = []
    for rep in range(2):
        prob = ctx.ba_problem(*_args(p))
        for again in range(2):
            if again:
                prob.reset()
            s = prob.run(capi.ba_default_options(max_solver_time_in_seconds=0.0))
            outs.append((s["num_iterations"], s["final_cost"]) + prob.download())
        prob.close()
    for o in outs[1:]:
        assert o[0] == outs[0][0] and o[1] == outs[0][1]
        assert np.array_equal(o[2], outs[0][2]) and np.array_equal(o[3], outs[0][3]) and o[4] == outs[0][4]


def test_many_cameras_take_the_atomics_path_and_agree(ctx, oracle):
    """1400 cameras: the per-(camera pair) partial blocks of the deterministic mode would need > 256 MB, so the solver switches to
    the atomics ("red") formulation by itself; the reduced system still matches the oracle."""
    p = synth.make_ba_problem(n_cams=1400, n_pts=3000, obs_per_pt=4, seed=31)
    prob = ctx.ba_problem(*_args(p))
    g = prob.reduced_system(1e4); o = oracle.ba_reduced_system(*_args(p), radius=1e4)
    np.testing.assert_allclose(g["S"], o["S"], rtol=0, atol=2e-11 * np.abs(o["S"]).max())
    np.testing.assert_allclose(g["rhs"], o["rhs"], rtol=0, atol=1e-10 * np.abs(o["rhs"]).max())
    prob.close()
