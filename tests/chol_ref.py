"""Extended-precision reference for the dense SPD solve of the bundle adjustment (csrc/chol.cuh, sfmb200_dense_spd_solve).

Everything is measured against the STORED double matrix, never the matrix a generator meant to build:
  * exact_residual(A, x, b): b - A x with every product split exactly (Veltkamp/Dekker) and each row summed by math.fsum;
  * reference_solve(A, b):   LAPACK (float64 Cholesky) plus rounds of iterative refinement on that exact residual, returned as
                             an unevaluated sum x + dx (dx = the next correction), good to well below one ulp of x;
  * factor_ratios(A, L):     |A - L L^T|_ij / (u (|L| |L^T|)_ij) in 80-bit long double, the componentwise backward error of a
                             Cholesky factor in units of the unit roundoff.  A factor computed in any summation order has
                             ratio_ij <= min(i, j) + 1 (+ O(u)) (Higham, Accuracy and Stability of Numerical Algorithms, 10.1).
Generators are seeded; each returns a symmetric matrix of which only the lower triangle matters.
"""
import math

import numpy as np
import scipy.linalg as sla

U = 2.0 ** -53
_SPLIT = 134217729.0            # 2^27 + 1


def longdouble_ok():
    return np.finfo(np.longdouble).nmant >= 63


# ------------------------------------------------------------------------------------------------------------- generators
def spd_cond(n, kappa, seed):
    """Q diag(sigma) Q^T, sigma geometric from 1 down to 1/kappa, Q Haar-random orthogonal."""
    rs = np.random.RandomState(seed)
    Q, R = np.linalg.qr(rs.standard_normal((n, n)))
    Q *= np.sign(np.diag(R))
    s = np.logspace(0, -math.log10(kappa), n) if n > 1 else np.ones(1)
    A = (Q * s) @ Q.T
    return np.tril(A) + np.tril(A, -1).T


def spd_graded(n, seed, lo=-140, hi=140):
    """D M D with M a well-conditioned SPD matrix (kappa 10) and D = diag(10^t), t spread over [lo, hi] in a random order."""
    rs = np.random.RandomState(seed + 7919)
    d = 10.0 ** rs.permutation(np.linspace(lo, hi, n))
    M = spd_cond(n, 10.0, seed)
    A = (d[:, None] * M) * d[None, :]
    return np.tril(A) + np.tril(A, -1).T


def spd_diag_dominant(n, seed):
    rs = np.random.RandomState(seed)
    B = rs.uniform(-1, 1, (n, n))
    A = np.tril(B, -1); A = A + A.T
    A[np.diag_indices(n)] = np.abs(A).sum(1) + rs.uniform(0.5, 1.5, n)
    return A


def negative_pivot(n, k, seed):
    """L D L^T with L unit lower triangular (entries of size 0.3) and D = 1 except D[k] = -1: pivots 0..k-1 are positive,
    pivot k is about -1."""
    rs = np.random.RandomState(seed)
    L = np.tril(rs.uniform(-0.3, 0.3, (n, n)), -1) + np.eye(n)
    d = np.ones(n); d[k] = -1.0
    A = (L * d) @ L.T
    return np.tril(A) + np.tril(A, -1).T


def zero_pivot(n, k, seed):
    """An SPD matrix with row and column k replaced by zeros: pivot k is exactly 0."""
    A = spd_diag_dominant(n, seed)
    A[k, :] = 0.0; A[:, k] = 0.0
    return A


def cond2(A):
    """2-norm condition number of the stored matrix (eigenvalues of its symmetric lower-triangle completion)."""
    S = np.tril(A) + np.tril(A, -1).T
    w = np.linalg.eigvalsh(S)
    return w[-1] / w[0]


# ------------------------------------------------------------------------------------------------------------- exact residual
def _split(a):
    c = _SPLIT * a
    hi = c - (c - a)
    return hi, a - hi


def two_prod(a, b):
    """p, e with p + e == a * b exactly (no overflow, no underflow in the error term)."""
    p = a * b
    ah, al = _split(a); bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def exact_residual(A, x, b):
    """b - A x for the symmetric matrix whose lower triangle A holds, each row's 2n + 1 terms summed exactly and rounded once."""
    S = np.tril(A) + np.tril(A, -1).T
    p, e = two_prod(S, x[None, :])
    terms = np.concatenate([b[:, None], -p, -e], axis=1)
    return np.array([math.fsum(row) for row in terms.tolist()])


# ------------------------------------------------------------------------------------------------------------- reference solve
def lapack_solve(A):
    S = np.tril(A) + np.tril(A, -1).T
    return sla.cho_factor(S, lower=True, check_finite=False)


def reference_solve(A, b, rounds=4, cf=None):
    """(x, dx): LAPACK's solution refined `rounds` times with the exact residual; dx = one more correction, not added, so that
    x + dx is the solution to about u^2 kappa relative."""
    cf = cf if cf is not None else lapack_solve(A)
    x = sla.cho_solve(cf, b, check_finite=False)
    for _ in range(rounds):
        x = x + sla.cho_solve(cf, exact_residual(A, x, b), check_finite=False)
    return x, sla.cho_solve(cf, exact_residual(A, x, b), check_finite=False)


def forward_error(xhat, ref):
    """||xhat - x||_inf / ||x||_inf with x = x0 + dx given as ref = (x0, dx)."""
    x0, dx = ref
    return np.max(np.abs((xhat - x0) - dx)) / np.max(np.abs(x0))


def backward_error(A, xhat, b):
    """Normwise backward error ||b - A xhat||_inf / (||A||_inf ||xhat||_inf + ||b||_inf), residual exact."""
    S = np.tril(A) + np.tril(A, -1).T
    r = exact_residual(A, xhat, b)
    return np.max(np.abs(r)) / (np.max(np.abs(S).sum(1)) * np.max(np.abs(xhat)) + np.max(np.abs(b)))


# ------------------------------------------------------------------------------------------------------------- factor check
def factor_ratios(A, L):
    """ratio_ij = |A - L L^T|_ij / (u (|L| |L^T|)_ij) on the lower triangle (0 where both vanish, inf where only the residual
    does not), in 80-bit long double: the products of two doubles carry 2^-11 u relative, far below what is measured."""
    Ll = np.tril(L).astype(np.longdouble)
    Al = np.tril(A).astype(np.longdouble)
    R = np.abs(Al - Ll @ Ll.T)
    D = np.abs(Ll) @ np.abs(Ll).T
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(D > 0, R / (np.longdouble(U) * D), np.where(R > 0, np.inf, 0.0))
    return np.tril(r).astype(np.float64)


def factor_excess(r):
    """max over the lower triangle of ratio_ij - (min(i, j) + 1): <= about 1 for any correctly computed factor."""
    n = r.shape[0]
    k = np.minimum.outer(np.arange(n), np.arange(n)) + 1.0
    return float(np.max(np.tril(r - k)))
