"""The extended-precision reference of the dense SPD solve (tests/chol_ref.py) against mpmath at 50 digits, and proof that its
checks catch a factor that is wrong by a dropped rank-1 term or by 4 ulp in one entry."""
import math

import numpy as np
import pytest
import scipy.linalg as sla

import chol_ref as cr

mpmath = pytest.importorskip("mpmath")


def _mp_solve(A, b):
    """The exact solution of the stored system to 50 digits, solved in the symmetrically diagonal-scaled form (a graded matrix
    looks singular to mpmath's pivot test otherwise)."""
    with mpmath.workdps(60):
        S = np.tril(A) + np.tril(A, -1).T
        n = S.shape[0]
        s = [1 / mpmath.sqrt(mpmath.mpf(float(S[i, i]))) for i in range(n)]
        M = mpmath.matrix(n, n)
        for i in range(n):
            for j in range(n):
                M[i, j] = mpmath.mpf(float(S[i, j])) * s[i] * s[j]
        y = mpmath.lu_solve(M, mpmath.matrix([mpmath.mpf(float(b[i])) * s[i] for i in range(n)]))
        return [y[i] * s[i] for i in range(n)]


@pytest.mark.parametrize("n,kind,seed", [(1, "cond", 0), (7, "cond", 1), (31, "cond", 2), (48, "cond", 3), (33, "graded", 4),
                                         (48, "dd", 5), (20, "graded", 6)])
def test_refined_solution_and_exact_residual_agree_with_mpmath(n, kind, seed):
    A = {"cond": lambda: cr.spd_cond(n, 1e10, seed), "graded": lambda: cr.spd_graded(n, seed, -60, 60),
         "dd": lambda: cr.spd_diag_dominant(n, seed)}[kind]()
    b = np.random.RandomState(seed + 100).standard_normal(n)
    x0, dx = cr.reference_solve(A, b)
    xs = _mp_solve(A, b)
    with mpmath.workdps(50):
        xm = np.array([float(v) for v in xs])
        # x0 + dx is the exact solution to far below one ulp of x0; x0 itself is correctly rounded up to one ulp
        err = max(abs(mpmath.mpf(float(x0[i])) + mpmath.mpf(float(dx[i])) - xs[i]) for i in range(n))
        assert float(err) <= 1e-3 * cr.U * np.max(np.abs(xm))
        assert np.all(np.abs(x0 - xm) <= 2 * np.spacing(np.abs(xm)))
        # the exact residual of a perturbed x is b - A x rounded once
        xp = x0 * (1 + 1e-9 * np.random.RandomState(seed).standard_normal(n))
        r = cr.exact_residual(A, xp, b)
        S = np.tril(A) + np.tril(A, -1).T
        for i in range(n):
            ri = mpmath.mpf(float(b[i])) - mpmath.fsum(mpmath.mpf(float(S[i, j])) * mpmath.mpf(float(xp[j])) for j in range(n))
            assert r[i] == float(ri)


@pytest.mark.parametrize("kappa", [1e1, 1e6, 1e10, 1e14])
def test_generators_reach_the_condition_they_claim(kappa):
    A = cr.spd_cond(96, kappa, 3)
    assert 0.5 * kappa < cr.cond2(A) < 2 * kappa
    G = cr.spd_graded(96, 3)
    d = np.sqrt(np.diag(G))
    assert d.max() / d.min() > 1e270 and np.all(np.isfinite(G))
    assert np.linalg.eigvalsh(cr.spd_diag_dominant(64, 1)).min() > 0


@pytest.mark.parametrize("k", [0, 1, 33, 63])
def test_non_spd_generators_put_the_bad_pivot_where_they_say(k):
    A = cr.negative_pivot(64, k, 2)
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.cholesky(A)
    if k:
        np.linalg.cholesky(A[:k, :k])           # the leading block is SPD
    Z = cr.zero_pivot(64, k, 2)
    assert np.all(Z[k] == 0) and np.all(Z[:, k] == 0)


@pytest.mark.skipif(not cr.longdouble_ok(), reason="needs an 80-bit long double")
@pytest.mark.parametrize("n,kind", [(40, "cond"), (100, "dd"), (70, "graded"), (96, "cond14")])
def test_factor_check_passes_lapack(n, kind):
    A = {"cond": lambda: cr.spd_cond(n, 1e6, 1), "dd": lambda: cr.spd_diag_dominant(n, 1), "graded": lambda: cr.spd_graded(n, 1, -50, 50),
         "cond14": lambda: cr.spd_cond(n, 1e14, 1)}[kind]()
    L = np.linalg.cholesky(np.tril(A) + np.tril(A, -1).T)
    r = cr.factor_ratios(A, L)
    assert np.all(np.isfinite(r))
    assert r.max() <= n + 1 and cr.factor_excess(r) <= 1.0, (r.max(), cr.factor_excess(r))


@pytest.mark.skipif(not cr.longdouble_ok(), reason="needs an 80-bit long double")
def test_factor_check_catches_a_dropped_rank1_term():
    """Tile (2, 1) of a 96 x 96 factor computed without the term of column 5 (tile column 0): the factor of A plus that term."""
    n = 96
    A = cr.spd_diag_dominant(n, 4)
    S = np.tril(A) + np.tril(A, -1).T
    L = np.linalg.cholesky(S)
    E = np.zeros_like(S)
    E[64:96, 32:64] = np.outer(L[64:96, 5], L[32:64, 5])
    L2 = np.linalg.cholesky(S + E + E.T)
    r = cr.factor_ratios(A, L2)
    assert r[64:96, 32:64].max() > 1e6 and cr.factor_excess(r) > 1e6
    assert cr.factor_excess(cr.factor_ratios(A, L)) <= 1.0


@pytest.mark.skipif(not cr.longdouble_ok(), reason="needs an 80-bit long double")
@pytest.mark.parametrize("i,j", [(0, 0), (1, 0), (1, 1), (2, 2), (40, 1), (70, 2)])
def test_factor_check_catches_one_entry_moved_by_4_ulp(i, j):
    """4 ulp in an entry that dominates the products it enters: a change of 4 to 8 u relative against an allowance of
    min(i, j) + 2 u.  (Deeper in the factor the same move is inside the rounding error that any summation order may commit, so
    no backward-error check can see it.)"""
    n = 96
    A = cr.spd_diag_dominant(n, 8)
    L = np.linalg.cholesky(np.tril(A) + np.tril(A, -1).T)
    L2 = L.copy()
    for _ in range(4):
        L2[i, j] = np.nextafter(L2[i, j], np.inf)
    assert cr.factor_excess(cr.factor_ratios(A, L)) <= 1.0
    assert cr.factor_excess(cr.factor_ratios(A, L2)) > 1.5


def test_backward_and_forward_error_measures():
    A = cr.spd_cond(64, 1e8, 5)
    b = np.random.RandomState(1).standard_normal(64)
    ref = cr.reference_solve(A, b)
    cf = cr.lapack_solve(A)
    x = sla.cho_solve(cf, b)
    assert cr.backward_error(A, ref[0], b) <= cr.U
    assert cr.backward_error(A, x, b) <= 64 * 4 * cr.U
    assert cr.forward_error(ref[0], ref) <= cr.U and 0 < cr.forward_error(x, ref) < 1e8 * 64 * cr.U
    # a perturbation of one component by 1e-10 is seen by both
    y = x.copy(); y[7] *= 1 + 1e-10
    assert cr.forward_error(y, ref) > 1e-12 and cr.backward_error(A, y, b) > 1e-13
