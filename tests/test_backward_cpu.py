"""The componentwise backward-error harness (backward.py) without a GPU: the sparse assembly against LUProblem.dense, the
reference meeting every bound on every input the GPU tests use (the oracle's factors, LAPACK and an extended-precision
LU, and a NumPy restatement of trsm_kernel's blocked algorithm with explicit 16 x 16 inverses), and mutations of the
oracle's factors that the bounds catch and the normwise rel_err check of the parity tests does not."""
import numpy as np
import pytest
import scipy.linalg as sl

import backward as bw
from oracle import oracle
from superlu_dist_b200 import hostlib
from test_gpu_kernels import lu_nopivot
from util import complex_problem, poisson_problem, rel_err


def test_assembly_matches_dense():
    prob, _ = poisson_problem(N=6, leaf=4, relax=8, maxsup=32)
    lay = prob.layers[0]
    assert np.array_equal(bw.panel_matrix(prob, lay).toarray(), prob.dense(lay, False))
    oracle.factor(prob)
    L, U = bw.factors(prob, lay)
    Ld, Ud = prob.dense(lay, True)
    assert np.array_equal(L.toarray(), Ld) and np.array_equal(U.toarray(), Ud)


@pytest.mark.parametrize("z", [False, True], ids=["d", "z"])
def test_ratio_counts_unreached_positions_as_infinite(z):
    prob = complex_problem(N=4, leaf=4, relax=8, maxsup=16) if z else poisson_problem(N=4, leaf=4, relax=8, maxsup=16)[0]
    F = bw.panel_matrix(prob, prob.layers[0])
    oracle.factor(prob)
    L, U = bw.factors(prob, prob.layers[0])
    assert bw.factor_ratio(F, L, U)[0] <= bw.factor_bound(prob)
    F = F.tolil()
    F[0, prob.n - 1] += 1.0     # no product of the factors reaches (0, n - 1) in this ordering
    assert (abs(L) @ abs(U))[0, prob.n - 1] == 0
    assert bw.factor_ratio(F.tocsr(), L, U)[0] == np.inf


# ------------------------------------------------------------------------------------------------------ kernel inputs
def _z_widths(z):
    return (bw.ZFAMILIES, bw.ZWIDTHS) if z else (bw.FAMILIES, bw.WIDTHS)


@pytest.mark.parametrize("z", [False, True], ids=["d", "z"])
@pytest.mark.parametrize("family", bw.ZFAMILIES)
def test_reference_kernels_meet_bounds(family, z):
    """Every (width, family) input of test_gpu_backward.py: the extended-precision LU and the same LU in double for the
    diagonal LU, LAPACK and the blocked-inverse restatement for both TRSM cases"""
    fams, widths = _z_widths(z)
    if family not in fams:
        pytest.skip("complex pivots are a doublecomplex family")
    dt = np.complex128 if z else np.float64
    for ns in widths:
        bound = bw.kernel_bound(ns, dt)
        m = bw.vecs_for(ns, family)
        a = bw.diag_lu_input(family, ns, 3, ns, z)
        out, tiny = bw.lu_nopivot_ld(a[:ns], bw.THRESH)
        r, rep = bw.diag_lu_ratio(a, np.vstack([out, a[ns:]]), bw.THRESH)
        assert r <= bound and rep == tiny, (ns, r, bound, rep, tiny)
        if family == "tiny":
            assert tiny == len([c for c in bw.TINY_COLS if c < ns])
        else:           # the same elimination in double: the input stays in range without the wider exponent
            r, _ = bw.diag_lu_ratio(a, np.vstack([lu_nopivot(a[:ns]), a[ns:]]))
            assert r <= bound, ("double LU", ns, r, bound)
        u, b = bw.trsm_l_input(family, ns, m, ns + 1, z)
        x = sl.solve_triangular(np.triu(u), b.T, trans="T", lower=False).T
        assert bw.trsm_l_ratio(u, b, x) <= bound, ("lapack L", ns)
        assert bw.trsm_l_ratio(u, b, bw.trsm_blocked(np.triu(u), b, False)) <= bound, ("blocked L", ns)
        if family in ("tiny", "zpivots"):
            continue          # a unit lower triangle has no pivots
        lo, b = bw.trsm_u_input(family, ns, m, ns + 2, z)
        lt = np.tril(lo, -1) + np.eye(ns)
        x = sl.solve_triangular(lt, b, lower=True, unit_diagonal=True)
        assert bw.trsm_u_ratio(lo, b, x) <= bound, ("lapack U", ns)
        assert bw.trsm_u_ratio(lo, b, bw.trsm_blocked(lt.T, b.T, True).T) <= bound, ("blocked U", ns)


@pytest.mark.parametrize("z", [False, True], ids=["d", "z"])
@pytest.mark.parametrize("family", bw.GEMM_FAMILIES)
def test_reference_gemm_meets_bound(family, z):
    for (m, n, k) in bw.GEMM_SHAPES:
        a, b, c = bw.gemm_input(family, m, n, k, m + n + k, z)
        assert bw.gemm_sub_ratio(a, b, c, c - a @ b) <= bw.gemm_bound(k, c.dtype), (m, n, k)


# ------------------------------------------------------------------------------------------- the oracle's factors
def _oracle_ratio(prob):
    F = bw.panel_matrix(prob, prob.layers[0])
    info, _, tiny = oracle.factor(prob)
    L, U = bw.factors(prob, prob.layers[0])
    r, rep = bw.factor_ratio(F, L, U, prob.thresh if prob.replace_tiny_pivot else None)
    return info, r, rep, tiny


@pytest.mark.parametrize("name", list(bw.PROBLEMS) + list(bw.ZPROBLEMS))
def test_oracle_factors_meet_bound(name):
    prob = complex_problem(**bw.ZPROBLEMS[name]) if name in bw.ZPROBLEMS else poisson_problem(**bw.PROBLEMS[name])[0]
    info, r, rep, tiny = _oracle_ratio(prob)
    assert info == 0 and rep == tiny == 0
    assert r <= bw.factor_bound(prob), (r, bw.factor_bound(prob))


def test_oracle_shifted_factors_meet_bound():
    from test_inertia_cpu import shifted
    prob, (rp, ci, v) = poisson_problem(**bw.SHIFT_KW)
    prob.fill_layer(0, rp, ci, shifted(rp, ci, v, bw.shift_sigma()))
    info, r, rep, tiny = _oracle_ratio(prob)
    d = bw.factors(prob, prob.layers[0])[1].diagonal()
    assert info == 0 and (d < 0).any() and (d > 0).any()
    assert r <= bw.factor_bound(prob)


def test_oracle_kkt_factors_with_replaced_pivots_meet_bound():
    from test_gpu_static_pivot import problem
    from test_static_pivot_cpu import scale_values
    prob, rp, ci, v, perm_r = problem(bw.kkt_matrix())
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    prob.fill_layer(0, *hostlib.row_permute(rp, ci, scale_values(v, rows, ci, R, Cs), perm_r))
    prob.replace_tiny_pivot, prob.thresh = 1, bw.KKT_THRESH
    info, r, rep, tiny = _oracle_ratio(prob)
    assert info == 0 and rep == tiny > 0
    assert r <= bw.factor_bound(prob)


# ------------------------------------------------------------------------------------------------------ mutations
@pytest.fixture(scope="module")
def oracle_factors():
    prob, _ = poisson_problem(N=10, leaf=8, relax=16, maxsup=128)
    F = bw.panel_matrix(prob, prob.layers[0])
    oracle.factor(prob)
    L, U = bw.factors(prob, prob.layers[0])
    return prob, F, L, U


def test_unperturbed_factors_pass(oracle_factors):
    prob, F, L, U = oracle_factors
    assert bw.factor_ratio(F, L, U)[0] <= bw.factor_bound(prob)


def test_one_l_entry_times_one_plus_1e12_fails_and_rel_err_misses_it(oracle_factors):
    """The entry whose product with its pivot dominates its column of |L| |U| the most (an L entry computed in a
    slightly wrong precision, or a lost low-order term)"""
    prob, F, L, U = oracle_factors
    lo = L.tocoo()
    strict = lo.row > lo.col
    r, c, v = lo.row[strict], lo.col[strict], lo.data[strict]
    D = (abs(L) @ abs(U)).tocsr()
    den = np.asarray(D[r, c]).ravel()
    share = np.where(den > 0, np.abs(v * U.diagonal()[c]) / np.where(den > 0, den, 1), 0)
    i = int(np.argmax(share))
    L2 = L.tolil()
    L2[r[i], c[i]] *= 1 + 1e-12
    L2 = L2.tocsr()
    assert bw.factor_ratio(F, L2, U)[0] > bw.factor_bound(prob)
    assert rel_err(L2.toarray(), L.toarray()) < 1e-10      # the parity tests' bar: passes


def test_one_small_fill_entry_of_u_zeroed_fails(oracle_factors):
    """A Schur scatter that drops the contributions to one small fill entry"""
    prob, F, L, U = oracle_factors
    uo = U.tocoo()
    keep = uo.col > uo.row
    r, c, v = uo.row[keep], uo.col[keep], uo.data[keep]
    fill = np.asarray(F[r, c]).ravel() == 0
    cand = np.nonzero(fill & (v != 0))[0]
    i = cand[np.argmin(np.abs(v[cand]))]
    assert abs(v[i]) < 1e-3 * abs(U).max()
    U2 = U.tolil()
    U2[r[i], c[i]] = 0.0
    assert bw.factor_ratio(F, L, U2.tocsr())[0] > bw.factor_bound(prob)


def test_one_panel_rounded_through_float32_fails(oracle_factors):
    prob, F, _, _ = oracle_factors
    lay = prob.layers[0].copy()
    k = int(np.argmax(prob.lval_len))
    lo, hi = lay.lval_off[k], lay.lval_off[k + 1]
    lay.lval[lo:hi] = lay.lval[lo:hi].astype(np.float32)
    L2, U2 = bw.factors(prob, lay)
    assert bw.factor_ratio(F, L2, U2)[0] > bw.factor_bound(prob)
