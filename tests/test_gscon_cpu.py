"""The NumPy restatement of LAPACK's dlacn2 / zlacn2 driven as dgecon / zgecon drive it, the oracle of the GPU condition
estimator (tests/test_gpu_gscon.py), checked here against scipy.linalg.lapack.dgecon / zgecon on getrf of the same matrix."""
import numpy as np
import pytest
import scipy.linalg as sl
import scipy.linalg.lapack as la

ITMAX = 5
SAFMIN = np.finfo(np.float64).tiny


def _sign(x, cplx):
    """dlacn2: +1 where x >= 0, else -1; zlacn2: x / |x|, or 1 where |x| <= safmin"""
    if not cplx:
        return np.where(x >= 0, 1.0, -1.0)
    a = np.abs(x)
    return np.where(a > SAFMIN, x / np.where(a > SAFMIN, a, 1.0), 1.0 + 0j)


def lacn2(solve, solve_t, n, cplx):
    """dlacn2 / zlacn2 step for step: estimate ||B||_1, where solve(v) = B v ("kase 1") and solve_t(v) = B^T v, B^H v
    in complex ("kase 2").  -> (est, number of solves)"""
    dt = np.complex128 if cplx else np.float64
    x = solve(np.full(n, 1.0 / n, dt))
    nsolves = 1
    if n == 1:
        return float(np.abs(x[0])), nsolves
    est = np.abs(x).sum()
    isgn = _sign(x, cplx)
    x = solve_t(isgn.copy())
    nsolves += 1
    j = int(np.argmax(np.abs(x)))                     # idamax / izmax1: the lowest index on a tie
    it = 2
    while True:
        e = np.zeros(n, dt)
        e[j] = 1.0
        x = solve(e)
        nsolves += 1
        estold, est = est, np.abs(x).sum()
        if not cplx and np.array_equal(_sign(x, cplx), isgn):
            break                                     # repeated sign vector: converged
        if est <= estold:
            break                                     # cycling
        isgn = _sign(x, cplx)
        x = solve_t(isgn.copy())
        nsolves += 1
        jlast, j = j, int(np.argmax(np.abs(x)))
        xl = np.abs(x[jlast]) if cplx else x[jlast]   # dlacn2 compares the signed entry
        if xl != np.abs(x[j]) and it < ITMAX:
            it += 1
            continue
        break
    i = np.arange(n)
    x = solve((np.where(i % 2 == 0, 1.0, -1.0) * (1.0 + i / (n - 1))).astype(dt))   # the alternating vector
    nsolves += 1
    temp = 2.0 * (np.abs(x).sum() / (3 * n))
    return float(max(est, temp)), nsolves


def gscon_dense(F, norm, anorm=None):
    """(rcond, est, solves) of the restatement on a dense F, as dgecon / zgecon: norm '1' estimates ||F^-1||_1 ('kase 1'
    solves with F, 'kase 2' with F^T / F^H), norm 'I' swaps the kases.  anorm defaults to ||F|| in that norm."""
    F = np.asarray(F)
    cplx = np.iscomplexobj(F)
    n = F.shape[0]
    lu = sl.lu_factor(F)
    plain = lambda v: sl.lu_solve(lu, v)                          # noqa: E731
    adj = lambda v: sl.lu_solve(lu, v, trans=2 if cplx else 1)    # noqa: E731
    one = norm in ("1", "O", "o")
    est, ns = lacn2(plain, adj, n, cplx) if one else lacn2(adj, plain, n, cplx)
    if anorm is None:
        anorm = np.abs(F).sum(axis=0 if one else 1).max()
    return (1.0 / est) / anorm, est, ns


def _matrix(n, cplx, seed):
    """A diagonally dominant matrix with a random sparse pattern (2 % dense), random signs and magnitudes"""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n)) * (rng.random((n, n)) < 0.02)
    if cplx:
        A = A + 1j * rng.standard_normal((n, n)) * (A != 0)
    A[np.diag_indices(n)] += np.abs(A).sum(1) * rng.uniform(0.3, 1.2, n) + 1e-3
    return A


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("norm", ["1", "I"])
@pytest.mark.parametrize("n,seed", [(300, 0), (500, 1), (800, 2)])
def test_restatement_matches_lapack_gecon(n, seed, norm, cplx):
    A = _matrix(n, cplx, seed)
    rc, est, ns = gscon_dense(A, norm)
    anorm = np.abs(A).sum(axis=0 if norm == "1" else 1).max()
    lu, _, info = (la.zgetrf if cplx else la.dgetrf)(A)
    assert info == 0
    ref, info = (la.zgecon if cplx else la.dgecon)(lu, anorm, norm=norm)
    assert info == 0
    assert abs(rc - ref) <= 1e-12 * ref, (rc, ref)
    assert 4 <= ns <= 11
    exact = np.abs(np.linalg.inv(A)).sum(axis=0 if norm == "1" else 1).max()
    assert est <= exact * (1 + 1e-12)


def test_restatement_exact_on_m_matrix():
    """For an inverse with nonnegative entries the kase-2 solve of the all-ones sign vector finds the heaviest column:
    the estimate is the exact norm."""
    n = 64
    A = 2.2 * np.eye(n) - np.eye(n, k=1) - np.eye(n, k=-1)
    _, est, _ = gscon_dense(A, "1")
    exact = np.abs(np.linalg.inv(A)).sum(axis=0).max()
    assert abs(est - exact) <= 1e-12 * exact


def test_restatement_order_one():
    rc, est, ns = gscon_dense(np.array([[4.0]]), "1")
    assert ns == 1 and est == 0.25 and rc == 1.0
