"""Bundle adjustment at the limits of the dense solve's launch set-up (K4, csrc/ba.cu: chol_setup): a problem past 1023 cameras,
whose one-CTA back substitution needs more than the 48 KB of shared memory a launch gets without opting in, and two live
problems of different sizes, where the second one created must not lower a shared-memory limit the first one launches with."""
import numpy as np
import pytest

import chol_ref as cr
from sfm_toy_library_b200 import capi, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _args(p):
    return p["cams"], p["pts"], p["focal"], p["obs_xy"], p["obs_cam"], p["pt_off"]


def test_more_than_1023_cameras_solve(ctx):
    """1100 cameras (n = 6601): the one-CTA back substitution keeps 8 x 6624 bytes of y in shared memory, past the 48 KB a
    launch gets without opting in.  Two LM iterations run and lower the cost, and the dense solve of the problem's own reduced
    system has a backward error within 4 n u of exact."""
    p = synth.make_ba_problem(n_cams=1100, n_pts=2200, obs_per_pt=3, seed=41)
    prob = ctx.ba_problem(*_args(p))
    g = prob.reduced_system(1e4)
    s = prob.run(capi.ba_default_options(max_num_iterations=2, max_solver_time_in_seconds=0.0))
    prob.close()
    assert s["num_iterations"] >= 1 and s["num_successful_steps"] >= 1 and s["final_cost"] < s["initial_cost"], s
    x, fail = ctx.dense_spd_solve(g["S"], g["rhs"])
    assert fail[0] == 0
    n = g["rhs"].shape[0]
    assert cr.backward_error(g["S"], x[0], g["rhs"]) <= 4 * n * cr.U


def _run_alone_and_together(ctx, pa, pb, opts):
    def res(prob):
        s = prob.run(opts)
        return (s["num_iterations"], s["final_cost"]) + prob.download()
    alone = []
    for p in (pa, pb):
        prob = ctx.ba_problem(*_args(p))
        alone.append(res(prob))
        prob.close()
    A = ctx.ba_problem(*_args(pa)); B = ctx.ba_problem(*_args(pb))     # the second, smaller problem is created last
    together = [res(A), res(B)]
    A.close(); B.close()
    for a, t in zip(alone, together):
        assert a[:2] == t[:2] and all(np.array_equal(u, v) for u, v in zip(a[2:4], t[2:4])) and a[4] == t[4]


def test_two_live_problems_keep_their_backsolve_shared_memory(ctx):
    """A 400-camera problem (cluster back substitution, ~176 KB of shared memory) and a 3-camera one created after it: each
    runs bitwise as it does alone."""
    opts = capi.ba_default_options(max_num_iterations=4, max_solver_time_in_seconds=0.0)
    _run_alone_and_together(ctx, synth.make_ba_problem(n_cams=400, n_pts=2000, obs_per_pt=4, seed=43),
                            synth.make_ba_problem(n_cams=3, n_pts=100, obs_per_pt=3, seed=44), opts)


def test_two_live_problems_keep_their_stored_z_backsub_shared_memory(ctx, monkeypatch):
    """The stored-Z back-substitution stages 144 bytes per camera: 280 cameras (40 KB) and then 220 cameras (31 KB) created
    while the first is alive; each runs bitwise as it does alone.  (Both also take the cluster back substitution, whose limit the
    second problem would lower as well.)"""
    monkeypatch.setenv("SFMB200_BA_BACKSUB", "stored")
    opts = capi.ba_default_options(max_num_iterations=4, max_solver_time_in_seconds=0.0)
    _run_alone_and_together(ctx, synth.make_ba_problem(n_cams=280, n_pts=2000, obs_per_pt=4, seed=45),
                            synth.make_ba_problem(n_cams=220, n_pts=2000, obs_per_pt=4, seed=46), opts)
