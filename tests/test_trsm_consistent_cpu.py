"""The panel TRSM on consistent right-hand sides (B = X T with moderate X) without a GPU: LAPACK and trsm_kernel's
algorithm with one correction step per 16-column block (backward.trsm_blocked, refine=1) meet the kernel bound on every
input of test_gpu_trsm_consistent.py, and the plain product with the explicit 16 x 16 inverse (refine=0) does not, so
the GPU tests can see that defect.  Then the planted factors and the indefinite shifts of the GPU tests: the oracle meets
the factorization bound, and the restated panel solves on its factors behave as on the dense inputs."""
import numpy as np
import pytest
import scipy.linalg as sl

import backward as bw
from oracle import oracle
from util import complex_problem, poisson_problem

CASES = [(z, ns, delta) for z in (False, True) for ns in (bw.ZCWIDTHS if z else bw.CWIDTHS) for delta in bw.DELTAS]


def l_case(ns, delta, z):
    return bw.trsm_l_consistent(ns, bw.CVECS, delta, bw.consistent_positions(ns), ns, z)


def u_case(ns, delta, z):
    return bw.trsm_u_consistent(ns, bw.CVECS, delta, bw.consistent_positions(ns), ns + 1, z)


def l_ratios(ns, delta, z):
    """-> (LAPACK, refine=0, refine=1) ratios over the kernel bound of X U = B"""
    u, b = l_case(ns, delta, z)
    bound = bw.kernel_bound(ns, u.dtype)
    x = sl.solve_triangular(u, b.T, trans="T", lower=False).T
    return [bw.trsm_l_ratio(u, b, y) / bound for y in (x, bw.trsm_blocked(u, b, False, 0), bw.trsm_blocked(u, b, False, 1))]


def u_ratios(ns, delta, z):
    """-> (LAPACK, refine=0, refine=1) ratios over the kernel bound of L X = B"""
    lo, b = u_case(ns, delta, z)
    bound = bw.kernel_bound(ns, lo.dtype)
    x = sl.solve_triangular(lo, b, lower=True, unit_diagonal=True)
    return [bw.trsm_u_ratio(lo, b, y) / bound for y in (x, bw.trsm_blocked(lo.T, b.T, True, 0).T,
                                                           bw.trsm_blocked(lo.T, b.T, True, 1).T)]


def test_positions_cover_first_middle_and_last_block():
    for ns in bw.CWIDTHS:
        pos = bw.consistent_positions(ns)
        nb = (ns + 15) // 16
        assert {p // 16 for p in pos} == {0, nb // 2, nb - 1}, (ns, pos)
        assert all(0 <= p < ns for p in pos)
    assert {p % 16 for ns in bw.CWIDTHS for p in bw.consistent_positions(ns) if p < ns - 1} >= {1, 7, 14}


@pytest.mark.parametrize("z", [False, True], ids=["d", "z"])
def test_lapack_and_refined_blocked_meet_bound(z):
    bad = []
    for zz, ns, delta in CASES:
        if zz != z:
            continue
        for case, rs in (("L", l_ratios(ns, delta, z)), ("U", u_ratios(ns, delta, z))):
            if not (rs[0] <= 1 and rs[2] <= 1):
                bad.append((case, ns, delta, rs[0], rs[2]))
    assert not bad, bad


# (case, z, ns, delta) where the unrefined product exceeds the bound, by the factor given (a margin below what it is)
UNREFINED_FAILS = [("L", False, 16, 1e-4, 100), ("L", False, 64, 1e-8, 1e5), ("L", False, 257, 1e-12, 1e8),
                   ("L", False, 512, 1e-8, 1e4), ("L", True, 33, 1e-4, 50), ("L", True, 256, 1e-12, 1e8),
                   ("U", False, 17, 1e-12, 100), ("U", False, 32, 1e-8, 10), ("U", False, 33, 1e-12, 3),
                   ("U", True, 17, 1e-12, 4), ("U", True, 31, 1e-8, 2)]


@pytest.mark.parametrize("case,z,ns,delta,factor", UNREFINED_FAILS)
def test_unrefined_product_with_inverse_exceeds_bound(case, z, ns, delta, factor):
    rs = (l_ratios if case == "L" else u_ratios)(ns, delta, z)
    assert rs[1] > factor, rs
    assert rs[0] <= 1 and rs[2] <= 1, rs


# ------------------------------------------------------------------------------------------------ planted factors
def planted_problem(name):
    if name in bw.ZPLANTED:
        return complex_problem(**bw.ZPLANTED[name])
    return poisson_problem(**bw.PLANTED[name])[0]


@pytest.mark.parametrize("name", list(bw.PLANTED) + list(bw.ZPLANTED))
def test_planted_factors(name):
    """F = fl(L0 U0) lands in the panels entry for entry; the oracle factors it without replacing pivots within the
    factorization bound (its ratio is the baseline of the GPU tests); the planted supernodes' panel solves, restated on
    the oracle's factors, exceed the kernel bound unrefined and meet it refined"""
    prob = planted_problem(name)
    F = bw.plant_factors(prob)
    assert (bw.panel_matrix(prob, prob.layers[0]) != F).nnz == 0
    nodes = bw.planted_nodes(prob)
    assert np.diff(np.asarray(prob.xsup))[nodes].max() == max(np.diff(np.asarray(prob.xsup)))
    prob.replace_tiny_pivot = 0
    info, _, tiny = oracle.factor(prob)
    L, U = bw.factors(prob, prob.layers[0])
    r, _ = bw.factor_ratio(F, L, U)
    assert info == 0 and tiny == 0
    assert r <= bw.factor_bound(prob), (r / bw.U, bw.factor_bound(prob) / bw.U)
    lr, ur = bw.panel_trsm_ratios(prob, L, U, 0, nodes)
    assert lr > 10, (lr, ur)
    lr, ur = bw.panel_trsm_ratios(prob, L, U, 1, nodes)
    assert lr <= 1 and ur <= 1, (lr, ur)


@pytest.mark.parametrize("sigma", ["gap", 283 / 64], ids=["shift_sigma", "283_64"])
def test_indefinite_shift_panels(sigma):
    """Poisson 12^3 - sigma I: the oracle within the factorization bound; the unrefined product with the inverse exceeds
    the kernel bound on the oracle's own L panels, the refined one does not (on every supernode)"""
    from test_inertia_cpu import shifted
    prob, (rp, ci, v) = poisson_problem(**bw.SHIFT_KW)
    prob.fill_layer(0, rp, ci, shifted(rp, ci, v, bw.shift_sigma() if sigma == "gap" else sigma))
    F = bw.panel_matrix(prob, prob.layers[0])
    info, _, _ = oracle.factor(prob)
    L, U = bw.factors(prob, prob.layers[0])
    assert info == 0 and bw.factor_ratio(F, L, U)[0] <= bw.factor_bound(prob)
    assert bw.panel_trsm_ratios(prob, L, U, 0)[0] > 2
    assert max(bw.panel_trsm_ratios(prob, L, U, 1)) <= 1
