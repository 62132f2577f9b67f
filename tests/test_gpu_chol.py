"""The dense SPD solve of the bundle adjustment (csrc/chol.cuh: dataflow tile Cholesky, cluster and one-CTA back substitutions) on
its own, through sfmb200_dense_spd_solve, against the extended-precision reference of tests/chol_ref.py.

Bounds (fixed from the error analysis, not from measurements):
  factor    |A - L L^T|_ij <= (n + 16) u (|L| |L^T|)_ij  whenever fail == 0 (n <= 700: the check runs in long double);
  forward   ||x - x*|| / ||x*|| <= max(10 x LAPACK's, n u kappa_1(A)), kappa_1 LAPACK's estimate (dpocon).  Ten times
            LAPACK's error alone is not a bound a backward-stable solve has to meet: the forward error of one solve is a draw
            anywhere below about kappa u, and LAPACK's own draw can be lucky (at n = 9, kappa = 1e6 this solve measured 19 x
            LAPACK's, and plain substitution with numpy's factor reaches 29 x LAPACK's on one of 40 such systems);
  backward  ||b - A x|| / (||A|| ||x|| + ||b||) <= max(10 x LAPACK's, 4 n u), residual exact.
"""
import re

import numpy as np
import pytest
import scipy.linalg as sla

import chol_ref as cr
from sfm_toy_library_b200 import capi, synth

pytestmark = pytest.mark.gpu
U = cr.U
WORST = {"factor ratio / (n + 16)": 0.0, "forward / bound": 0.0, "backward / bound": 0.0, "forward": 0.0, "backward": 0.0,
         "factor ratio": 0.0}


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def max_grid(ctx):
    """The co-resident CTA count of the factorisation, read from the refusal of a larger grid."""
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.dense_spd_solve(np.eye(64), np.ones(64), grid=1 << 20)
    return int(re.search(r"exceeds the (\d+) co-resident", str(e.value)).group(1))


def cluster_fits(n):
    nb = (n - 1) // 32 + 1
    nwork = 32 * ((nb + 7) // 8)
    return 8 * (8 * 32 + 32 * 32 + nwork + 2 * 32 * nwork) <= 200 * 1024 and nwork + 32 <= 512


def paths(n):
    return (1, 2) if cluster_fits(n) else (2,)


def check_solution(A, b, x, rounds=4):
    n = b.shape[0]
    cf = cr.lapack_solve(A)
    ref = cr.reference_solve(A, b, rounds, cf)
    xl = sla.cho_solve(cf, b, check_finite=False)
    fe, fe_l = cr.forward_error(x, ref), cr.forward_error(xl, ref)
    be, be_l = cr.backward_error(A, x, b), cr.backward_error(A, xl, b)
    S = np.tril(A) + np.tril(A, -1).T
    rcond, info = sla.lapack.dpocon(cf[0], np.abs(S).sum(0).max(), uplo="L")
    fb, bb = max(10 * fe_l, n * U / rcond if rcond > 0 else np.inf), max(10 * be_l, 4 * n * U)
    WORST["forward"] = max(WORST["forward"], fe); WORST["backward"] = max(WORST["backward"], be)
    WORST["forward / bound"] = max(WORST["forward / bound"], fe / fb); WORST["backward / bound"] = max(WORST["backward / bound"], be / bb)
    assert np.all(np.isfinite(x))
    assert fe <= fb, f"n={n}: forward error {fe:.3e} > {fb:.3e} (LAPACK {fe_l:.3e})"
    assert be <= bb, f"n={n}: backward error {be:.3e} > {bb:.3e} (LAPACK {be_l:.3e})"


def check_factor(A, L):
    n = A.shape[0]
    if n > 700 or not cr.longdouble_ok():
        return
    r = cr.factor_ratios(A, L)
    WORST["factor ratio"] = max(WORST["factor ratio"], float(r.max()))
    WORST["factor ratio / (n + 16)"] = max(WORST["factor ratio / (n + 16)"], float(r.max()) / (n + 16))
    assert r.max() <= n + 16, f"n={n}: factor ratio {r.max():.2f} at {np.unravel_index(np.argmax(r), r.shape)}"


def solve_all(ctx, As, bs, rounds=4, grid=0):
    """Every back substitution that can run at this n: same factor bit for bit, each x within the bounds."""
    n = As.shape[-1]
    res = []
    for bsv in paths(n):
        x, L, fail = ctx.dense_spd_solve(As, bs, grid=grid, backsolve=bsv, want_L=True)
        assert np.all(fail == 0), (n, bsv, fail)
        res.append((x, L))
    for x, L in res[1:]:
        assert np.array_equal(L, res[0][1])
    for k in range(As.shape[0]):
        check_factor(As[k], res[0][1][k])
        for x, _ in res:
            check_solution(As[k], bs[k], x[k], rounds)
    return res


def families(n, seed):
    kappa = [1e1, 1e6, 1e10, 1e14][seed % 4]
    As = np.stack([cr.spd_cond(n, kappa, seed), cr.spd_graded(n, seed, -40, 40), cr.spd_diag_dominant(n, seed)])
    bs = np.random.RandomState(seed + 1).standard_normal((3, n))
    return As, bs


@pytest.mark.parametrize("n", list(range(1, 71)))
def test_every_small_n(ctx, n):
    solve_all(ctx, *families(n, n))


@pytest.mark.parametrize("n", list(range(240, 272)))
def test_every_n_mod_32_around_eight_tiles(ctx, n):
    solve_all(ctx, *families(n, n))


@pytest.mark.parametrize("nc", [100, 180, 469, 470])
def test_ba_sizes(ctx, nc):
    """n = 6 nc + 1 (nc <= 12 are in the small-n sweep; nc = 5 puts the right-hand side in the last row of a tile)."""
    n = 6 * nc + 1
    A = cr.spd_cond(n, 1e8, nc)[None]
    b = np.random.RandomState(nc).standard_normal((1, n))
    solve_all(ctx, A, b, rounds=2)


@pytest.mark.parametrize("n", [607, 608, 609, 640, 641, 672, 673, 1500])
def test_one_cta_worker_boundary_and_more_tasks_than_ctas(ctx, n):
    """608 workers of the one-CTA back substitution own the columns left of the block; from n = 1500 (1082 tasks) the dataflow
    kernel has more tasks than co-resident CTAs."""
    A = cr.spd_cond(n, 1e6, n)[None]
    b = np.random.RandomState(n).standard_normal((1, n))
    solve_all(ctx, A, b, rounds=2)


@pytest.mark.parametrize("nb", [1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17])
def test_cluster_block_counts(ctx, nb):
    for n in (32 * nb - 3, 32 * nb):
        A = cr.spd_diag_dominant(n, nb)[None]
        b = np.random.RandomState(nb).standard_normal((1, n))
        solve_all(ctx, A, b, rounds=2)


def test_cluster_limit(ctx):
    for n in (2816, 2817):
        A = cr.spd_cond(n, 1e4, n)[None]
        b = np.random.RandomState(n).standard_normal((1, n))
        assert paths(n) == ((1, 2) if n == 2816 else (2,))
        solve_all(ctx, A, b, rounds=1)
    with pytest.raises(capi.SfmB200Error, match="cluster"):
        ctx.dense_spd_solve(A, b, backsolve=1)


def test_past_48kb_of_backsolve_shared_memory(ctx):
    """n = 6200: y needs 8 x 6208 bytes of shared memory in the one-CTA back substitution, past the 48 KB a launch gets without
    opting in (the size of a 1034-camera problem)."""
    n = 6200
    A = cr.spd_diag_dominant(n, 3)[None]
    b = np.random.RandomState(3).standard_normal((1, n))
    x, fail = ctx.dense_spd_solve(A, b)
    assert fail[0] == 0
    check_solution(A[0], b[0], x[0], rounds=1)


@pytest.mark.parametrize("nc,radius", [(40, 1e4), (40, 1e16), (100, 1e4), (100, 1e16)])
def test_reduced_systems_of_ba_problems(ctx, nc, radius):
    """The systems the LM loop solves; at radius 1e16 the LM diagonal vanishes and the gauge freedom leaves them nearly singular."""
    p = synth.make_ba_problem(n_cams=nc, n_pts=40 * nc, obs_per_pt=4, seed=nc)
    prob = ctx.ba_problem(p["cams"], p["pts"], p["focal"], p["obs_xy"], p["obs_cam"], p["pt_off"])
    g = prob.reduced_system(radius)
    prob.close()
    solve_all(ctx, g["S"][None], g["rhs"][None])


def test_scheduling_does_not_change_bits(ctx, max_grid):
    for n in (300, 1500):
        As, bs = families(n, 5)
        ref = ctx.dense_spd_solve(As, bs, want_L=True)
        for grid in (1, 2, 3, 7, max_grid):
            x, L, fail = ctx.dense_spd_solve(As, bs, grid=grid, want_L=True)
            assert np.all(fail == 0) and np.array_equal(x, ref[0]) and np.array_equal(L, ref[1]), (n, grid)


def test_consecutive_solves_do_not_interfere(ctx):
    for n in (31, 200, 1100):
        A1, A2 = cr.spd_cond(n, 1e6, 1), cr.spd_diag_dominant(n, 2)
        b1, b2 = np.random.RandomState(3).standard_normal((2, n))
        x, L, fail = ctx.dense_spd_solve(np.stack([A1, A2, A1]), np.stack([b1, b2, b1]), want_L=True)
        s1 = ctx.dense_spd_solve(A1, b1, want_L=True); s2 = ctx.dense_spd_solve(A2, b2, want_L=True)
        assert np.all(fail == 0)
        for k, s in ((0, s1), (1, s2), (2, s1)):
            assert np.array_equal(x[k], s[0][0]) and np.array_equal(L[k], s[1][0]), (n, k)


def test_only_the_lower_triangle_is_read(ctx):
    for n in (45, 300):
        As, bs = families(n, 9)
        ref = ctx.dense_spd_solve(As, bs, want_L=True)
        An = As.copy()
        iu = np.triu_indices(n, 1)
        for k in range(3):
            An[k][iu] = np.nan
        x, L, fail = ctx.dense_spd_solve(An, bs, want_L=True)
        assert np.all(fail == 0) and np.array_equal(x, ref[0]) and np.array_equal(L, ref[1])


@pytest.mark.parametrize("n", [40, 100, 130])
def test_non_spd_is_reported(ctx, n):
    """A negative pivot in the column-0 task and in merged tasks, then the context solves on as before."""
    b = np.ones(n)
    A0 = cr.spd_diag_dominant(n, 1)
    before = ctx.dense_spd_solve(A0, b, want_L=True)
    for k in sorted({0, 1, 2, 3, 31, 32, 33, 34, n - 1}):
        if k >= n:
            continue
        for A in (cr.negative_pivot(n, k, k), cr.zero_pivot(n, k, k)):
            for bsv in paths(n):
                x, fail = ctx.dense_spd_solve(A, b, backsolve=bsv)
                assert 0 < fail[0] < 1000, (n, k, bsv, fail)
    after = ctx.dense_spd_solve(A0, b, want_L=True)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])


@pytest.mark.parametrize("val", [np.nan, np.inf, -np.inf])
def test_non_finite_lower_triangle_is_reported(ctx, val):
    n = 100
    for (i, j) in [(0, 0), (5, 2), (40, 3), (99, 98), (99, 99), (64, 64), (70, 33)]:
        A = cr.spd_diag_dominant(n, 4)
        A[i, j] = val
        x, fail = ctx.dense_spd_solve(A, np.ones(n))
        assert 0 < fail[0] < 1000, (i, j, val, fail)


def _finite_or_failed(ctx, A, b):
    n = b.shape[0]
    for bsv in paths(n):
        x, fail = ctx.dense_spd_solve(A, b, backsolve=bsv)
        assert fail[0] < 1000
        if fail[0] == 0:
            check_solution(A, b, x[0])
    return fail[0]


def test_subnormal_pivot_and_minor_are_reported(ctx):
    """rsqrt.approx.ftz flushes a subnormal pivot or 2x2 minor to zero and returns +inf: the factor must not come back
    non-finite with fail == 0.  An overflowing minor (pivots ~1e160) makes an SPD matrix unsolvable here: it must fail.  A
    pivot of 1e200 whose minors stay in range solves.  A bad pivot early in the matrix turns every later pivot into NaN, which
    is caught anyway; only the last pivots of the matrix (n - 1, and the pair n - 2, n - 1) show whether the test itself holds."""
    n = 40
    for idx, d, pair, must_fail in [(n - 1, 1e-310, False, True), (n - 2, 1e-155, True, True), (n - 1, 1e200, False, False),
                                    (0, 1e-310, False, True), (5, 1e-310, False, True), (0, 1e-155, True, True), (2, 1e-155, True, True),
                                    (6, 1e-160, True, True), (0, 1e160, True, True), (3, 1e200, False, False)]:
        diag = np.ones(n)
        diag[idx] = d
        if pair:
            diag[idx + 1] = d                    # the pair's minor D2 = d^2: subnormal, or infinite
        A = np.diag(diag)
        b = diag * np.linspace(1, 2, n)         # x = linspace(1, 2): finite
        fail = _finite_or_failed(ctx, A, b)
        assert (fail != 0) == must_fail, (idx, d, fail)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("n", [33, 64, 100])
def test_graded_extremes_solve_or_fail(ctx, n, seed):
    """D M D with D from 1e-140 to 1e140: products of pivots leave the double range, so the solve fails or is right."""
    A = cr.spd_graded(n, seed, -140, 140)
    b = np.random.RandomState(seed).standard_normal(n) * np.sqrt(np.diag(A))
    _finite_or_failed(ctx, A, b)
    A = cr.spd_graded(n, seed, -70, 70)                        # pivots within [1e-140, 1e140]: must solve
    b = np.random.RandomState(seed).standard_normal(n) * np.sqrt(np.diag(A))
    x, fail = ctx.dense_spd_solve(A, b)
    assert fail[0] == 0
    check_solution(A, b, x[0])


def test_refusals(ctx, max_grid):
    A = np.eye(8); b = np.ones(8)
    for kw in (dict(grid=max_grid + 1), dict(grid=-1), dict(backsolve=3)):
        with pytest.raises(capi.SfmB200Error):
            ctx.dense_spd_solve(A, b, **kw)
    x, fail = ctx.dense_spd_solve(A, b, grid=max_grid)
    assert fail[0] == 0 and np.abs(x[0] - b).max() <= 4 * U


def test_zz_report_worst_measured(capsys):
    with capsys.disabled():
        print("\n[dense SPD solve, H100] worst measured: " + ", ".join(f"{k} {v:.3g}" for k, v in WORST.items()))
