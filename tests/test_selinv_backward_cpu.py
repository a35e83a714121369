"""Selected inversion step by step without a GPU: every step of every supernode solves its own equations to working
precision (backward.selinv_ratios, extended-precision residuals of H as returned) for oracle/selinv.py (substitution)
and for the sweep of slu_selinv.cu restated with its explicit 16 x 16 block inverses and one correction step
(backward.selinv_blocked, refine=1), on planted factors with small pivots, indefinite shifts, a KKT matrix with
replaced pivots and the selected-inversion fixtures.  The plain product with the block inverses (refine=0) fails on a
named subset, so the GPU tests can see that defect; the normwise checks against a dense inverse cannot.  Then the
log-determinant of the oracle against an exact sum of the pivots' logs."""
import functools

import numpy as np
import pytest

import backward as bw
from oracle import oracle, selinv
from superlu_dist_b200 import hostlib
from test_gpu_solve_trans import unsym_values
from test_scaled_parity import mixed_values
from test_trsm_consistent_cpu import planted_problem
from util import load_fixture, poisson_problem

SHIFTS = {"shift_gap": None, "shift_283_64": 283 / 64}
FIXTURES = ["g4_pddrive3d", "unsym360_mmd"]
GENERATED = {"poisson8_unsym": (dict(N=8, leaf=4, relax=8, maxsup=32), "unsym"),
             "fem5_mixed": (dict(N=5, leaf=4, relax=8, maxsup=200, fem=3), "mixed"),
             "poisson10_mixed": (dict(N=10, leaf=8, relax=16, maxsup=128), "mixed")}
# fem6_replaced: the planted pivots of fem6 at 1e-10, replaced under a threshold of 1e-8 (in-block offsets 1, 7, 14)
REPLACED = ("kkt", "fem6_replaced")
INPUTS = list(bw.PLANTED) + list(bw.ZPLANTED) + list(SHIFTS) + list(REPLACED) + FIXTURES + list(GENERATED)


def unfactored(name):
    """-> prob with layer 0 holding F = P A P^T, unfactored (replace_tiny_pivot and thresh set for REPLACED)"""
    if name in bw.PLANTED or name in bw.ZPLANTED:
        prob = planted_problem(name)
        bw.plant_factors(prob)
        prob.replace_tiny_pivot = 0
    elif name == "fem6_replaced":
        from test_gpu_trsm_consistent import REPLACE_DELTA, REPLACE_THRESH
        prob = planted_problem("fem6")
        bw.plant_factors(prob, REPLACE_DELTA)
        prob.replace_tiny_pivot, prob.thresh = 1, REPLACE_THRESH
    elif name in SHIFTS:
        from test_inertia_cpu import shifted
        prob, (rp, ci, v) = poisson_problem(**bw.SHIFT_KW)
        prob.fill_layer(0, rp, ci, shifted(rp, ci, v, bw.shift_sigma() if SHIFTS[name] is None else SHIFTS[name]))
    elif name == "kkt":
        from test_gpu_static_pivot import problem
        from test_static_pivot_cpu import scale_values
        prob, rp, ci, v, perm_r = problem(bw.kkt_matrix())
        _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        prob.fill_layer(0, *hostlib.row_permute(rp, ci, scale_values(v, rows, ci, R, Cs), perm_r))
        prob.replace_tiny_pivot, prob.thresh = 1, bw.KKT_THRESH
    elif name in FIXTURES:
        prob = load_fixture(name)[0]
    else:
        kw, values = GENERATED[name]
        prob, (rp, ci, v) = poisson_problem(**kw)
        prob.fill_layer(0, rp, ci, unsym_values(rp, ci, v) if values == "unsym" else mixed_values(rp, ci, v, seed=3))
    return prob


@functools.lru_cache(maxsize=None)
def factored(name):
    """-> prob with the oracle's factors in layer 0 (cached: the tests only read it)"""
    prob = unfactored(name)
    info, _, tiny = oracle.factor(prob)
    assert info == 0
    assert (tiny > 0) == (name in REPLACED), tiny
    return prob


@functools.lru_cache(maxsize=None)
def ratios(name, how):
    """-> (ratio / bound, ratio) of each step for H from 'oracle', 'refine0' or 'refine1' on the oracle's factors"""
    prob = factored(name)
    lay = prob.layers[0]
    hl, hu = selinv.selinv(prob, lay) if how == "oracle" else bw.selinv_blocked(prob, lay, int(how[-1]))
    return bw.selinv_ratios(prob, lay, hl, hu)


def report(name, how):
    s, r = ratios(name, how)
    return {step: f"{q:.3g} of the bound ({x / bw.U:.3g} u)" for step, q, x in zip(bw.SELINV_STEPS, s, r)}


@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("how", ["oracle", "refine1"])
def test_substitution_and_refined_blocked_meet_bounds(name, how):
    assert ratios(name, how)[0].max() <= 1, report(name, how)


# (input, step) where the plain product with the explicit block inverses exceeds its bound, by the factor given (a margin
# below what it is): the rows of H(R,K) solved against the planted (or replaced) small pivots of U_KK.  The other pairs
# are printed, not asserted: the indefinite shifts and the KKT matrix stay within their bounds, and H(K,C) of fem6,
# fem6_replaced and z200 is within a few tens of percent of its bound either way.
REFINE0_FAILS = {("top256", "H(R,K)"): 2, ("fem6", "H(R,K)"): 10, ("z200", "H(R,K)"): 5, ("fem6_replaced", "H(R,K)"): 100}


def test_unrefined_blocked_fails_on_the_named_inputs(capsys):
    seen = {}
    for name in INPUTS:
        s = ratios(name, "refine0")[0]
        for step, q in zip(bw.SELINV_STEPS, s):
            if q > 1:
                seen[(name, step)] = q
    with capsys.disabled():
        print("\nselinv with the explicit 16 x 16 inverses and no correction step exceeds the bound on: " +
              (", ".join(f"{n} {st} ({q:.3g} x)" for (n, st), q in sorted(seen.items())) if seen else "none"))
    for key, factor in REFINE0_FAILS.items():
        assert seen.get(key, 0) > factor, (key, seen)


def test_ratios_see_a_stray_and_a_missed_write():
    """One entry of H(K,C) off by 1e-10 relative, then one set to zero: both exceed the bound by far"""
    prob = factored("fem6")
    lay = prob.layers[0]
    hl, hu = selinv.selinv(prob, lay)
    q = int(np.argmax(np.abs(hu)))
    for v in (hu[q] * (1 + 1e-10), 0.0):
        h2 = hu.copy()
        h2[q] = v
        assert bw.selinv_ratios(prob, lay, hl, h2)[0][1] > 1e3


@pytest.mark.parametrize("name", INPUTS)
def test_oracle_logdet_against_exact_sum(name):
    from test_selinv_complex_cpu import complex_logdet
    prob = factored(name)
    lay = prob.layers[0]
    sign, la, tol, ptol = bw.pivot_logdet(prob, lay)
    s2, l2 = complex_logdet(prob, lay) if np.iscomplexobj(lay.lval) else selinv.logdet(prob, lay)
    assert abs(l2 - la) <= tol, (l2, la, tol)
    if np.iscomplexobj(lay.lval):
        assert abs(s2 - sign) <= ptol, (s2, sign, ptol)
    else:
        assert s2 == sign
