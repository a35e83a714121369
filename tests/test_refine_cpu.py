"""The NumPy restatement of slu_b200_gsrfs, the oracle of tests/test_gpu_refine.py: the device residual in its exact
operation order (residual_rows), pdgsrfs's refinement loop and LAPACK dgerfs's forward error bound driven by the dlacn2
restatement of tests/test_gscon_cpu.py.  Checked here against scipy.linalg.lapack.dgesvx / zgesvx (fact='N': getrf, getrs,
then dgerfs / zgerfs with ITMAX 5) on the same getrf factors."""
import numpy as np
import pytest
import scipy.linalg as sl
import scipy.linalg.lapack as la
import scipy.sparse as sp

from test_gscon_cpu import lacn2

EPS = np.finfo(np.float64).eps / 2          # dmach("Epsilon")
SAFMIN = np.finfo(np.float64).tiny          # dmach("Safe minimum")
ITMAX = 20                                  # pdgsrfs.c


def abs1(v):
    """|v|, cabs1 (|re| + |im|) for complex"""
    v = np.asarray(v)
    return np.abs(v.real) + np.abs(v.imag) if np.iscomplexobj(v) else np.abs(v)


def residual_rows(rp, ci, av, x, b):
    """(r, w) = (b - A x, |A| |x| + |b|) for one column, as refine_residual_kernel computes them: each row walks its
    entries in CSR order, every product and sum rounded on its own (complex products: four products, two sums), vectorised
    over the rows"""
    n = len(rp) - 1
    lens = np.diff(rp)
    cplx = np.iscomplexobj(av) or np.iscomplexobj(x) or np.iscomplexobj(b)
    re, im, w = np.zeros(n), np.zeros(n), np.zeros(n)
    for k in range(int(lens.max()) if n else 0):
        rows = np.nonzero(lens > k)[0]
        p = rp[rows] + k
        a, xv = av[p], x[ci[p]]
        if cplx:
            a, xv = a.astype(np.complex128), xv.astype(np.complex128)
            re[rows] = re[rows] + (a.real * xv.real - a.imag * xv.imag)
            im[rows] = im[rows] + (a.real * xv.imag + a.imag * xv.real)
        else:
            re[rows] = re[rows] + a * xv
        w[rows] = w[rows] + abs1(a) * abs1(xv)
    if cplx:
        b = b.astype(np.complex128)
        r = (b.real - re) + 1j * (b.imag - im)
    else:
        r = b - re
    return r, w + abs1(b)


def safe(n):
    safe1 = (n + 1) * SAFMIN
    return safe1, safe1 / EPS


def berr_of(r, w):
    """max_i |r_i| / w_i, (safe1 + |r_i|) / w_i where w_i <= safe2, rows with w_i = 0 skipped (pdgsrfs.c:214-230)"""
    safe1, safe2 = safe(len(r))
    ar = abs1(r)
    nz = w != 0
    s = np.where(w > safe2, ar / np.where(nz, w, 1.0), (safe1 + ar) / np.where(nz, w, 1.0))
    return float(s[nz].max()) if nz.any() else 0.0


def ferr_weights(r, w):
    """dgerfs's W_i = |r_i| + (n + 1) eps w_i, + safe1 where w_i <= safe2"""
    safe1, safe2 = safe(len(r))
    W = abs1(r) + ((len(r) + 1) * EPS) * w
    return np.where(w > safe2, W, W + safe1)


def gsrfs(rp, ci, av, b, x, solve, solve_h=None, itmax=ITMAX):
    """pdgsrfs's loop for one column (solve(v) = A^-1 v), then, with solve_h(v) = A^-T v (A^-H v in complex), dgerfs's
    forward error bound.  -> (x, berr, steps, ferr or None)"""
    x = np.array(x, copy=True)
    lstres, count = 3.0, 0
    while True:
        r, w = residual_rows(rp, ci, av, x, b)
        berr = berr_of(r, w)
        if not (berr > EPS and 2 * berr <= lstres and count < itmax):
            break
        x = x + solve(r)
        lstres, count = berr, count + 1
    if solve_h is None:
        return x, berr, count, None
    W = ferr_weights(r, w)
    cplx = np.iscomplexobj(av) or np.iscomplexobj(b)
    est, _ = lacn2(lambda v: W * solve_h(v), lambda v: solve(W * v), len(b), cplx)
    xm = abs1(x).max()
    return x, berr, count, (est / xm if xm != 0 else est)


def _dense(n, cplx, seed, cond=1e6):
    """A dense matrix with singular values spread over `cond` (so that refinement and the bound have work to do)"""
    rng = np.random.default_rng(seed)
    g = lambda: rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cplx else 0)   # noqa: E731
    U, _ = np.linalg.qr(g())
    V, _ = np.linalg.qr(g())
    return (U * np.logspace(0, -np.log10(cond), n)) @ V.conj().T


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("n,seed", [(60, 0), (150, 1), (300, 2)])
def test_restatement_matches_lapack_gesvx(n, seed, cplx):
    A = _dense(n, cplx, seed)
    rng = np.random.default_rng(seed + 10)
    b = rng.standard_normal(n) + (1j * rng.standard_normal(n) if cplx else 0)
    out = (la.zgesvx if cplx else la.dgesvx)(A, b[:, None], fact="N")
    x_ref, ferr_ref, berr_ref, info = out[7][:, 0], out[9][0], out[10][0], out[11]
    assert info == 0
    lu = sl.lu_factor(A)
    S = sp.csr_matrix(A)
    x, berr, steps, ferr = gsrfs(S.indptr, S.indices, S.data, b, sl.lu_solve(lu, b), lambda v: sl.lu_solve(lu, v),
                                 lambda v: sl.lu_solve(lu, v, trans=2 if cplx else 1), itmax=5)
    assert berr <= 4 * EPS and berr_ref <= 4 * EPS, (berr, berr_ref)
    assert abs(ferr - ferr_ref) <= 0.05 * ferr_ref, (ferr, ferr_ref)
    assert 0 <= steps <= 5
    assert np.abs(x - x_ref).max() <= 10 * ferr * np.abs(x).max()


def test_zero_column_and_zero_start():
    A = sp.csr_matrix(_dense(40, False, 3, cond=10.0))
    lu = sl.lu_factor(A.toarray())
    solve = lambda v: sl.lu_solve(lu, v)   # noqa: E731
    z = np.zeros(40)
    x, berr, steps, _ = gsrfs(A.indptr, A.indices, A.data, z, z, solve)
    assert berr == 0.0 and steps == 0 and np.array_equal(x, z)
    b = np.random.default_rng(4).standard_normal(40)
    _, berr0, steps0, _ = gsrfs(A.indptr, A.indices, A.data, b, z, solve, itmax=0)
    assert berr0 == 1.0 and steps0 == 0
    x, berr, steps, _ = gsrfs(A.indptr, A.indices, A.data, b, z, solve)
    assert steps >= 1 and berr <= 4 * EPS


def test_residual_rows_order():
    """the CSR order of a row decides the rounding: a row whose partial sums cancel differs from its sorted sum"""
    rp = np.array([0, 3])
    ci = np.array([0, 1, 2])
    av = np.array([1.0, 1e16, -1e16])
    r, w = residual_rows(rp, ci, av, np.ones(3), np.zeros(1))
    assert r[0] == -((1.0 + 1e16) - 1e16) and w[0] == (1.0 + 1e16) + 1e16
