"""oracle/selinv.py, the NumPy restatement of slu_b200_selinv: H = F^-T at every stored position of L + U against a dense
inverse of the oracle's own factors, and its log-determinant against numpy.linalg.slogdet."""
import numpy as np
import pytest

from oracle import oracle, selinv
from test_gpu_solve_trans import unsym_values
from test_scaled_parity import mixed_values, panel_coords
from util import load_fixture, poisson_problem

TOL = 1e-10
FIXTURES = ["g4_pddrive3d", "g20_pddrive3d", "poisson8_nd", "poisson12_nd_tiny", "fem5_mmd", "unsym360_mmd"]
GENERATED = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=5, leaf=4, relax=8, maxsup=200, fem=3),
             dict(N=10, leaf=8, relax=16, maxsup=128)]


def check_against_dense(prob, lay):
    """H from the oracle against inv(L U)^T at every stored position: within TOL max |F^-1|, diagonal within TOL relative"""
    L, U = prob.dense(lay, True)
    G = np.linalg.inv(L @ U)
    hl, hu = selinv.selinv(prob, lay)
    lrow, lcol, urow, ucol = panel_coords(prob, lay)
    scale = np.abs(G).max()
    assert (lrow >= 0).all()
    assert np.abs(hl - G.T[lrow, lcol]).max() <= TOL * scale
    u = urow >= 0                                   # a problem without U panels has a one-element placeholder arena
    assert np.abs(hu[u] - G.T[urow[u], ucol[u]]).max(initial=0.0) <= TOL * scale
    dg = lrow == lcol
    d = G[lrow[dg], lcol[dg]]
    assert dg.sum() == prob.n
    assert (np.abs(hl[dg] - d) <= TOL * np.abs(d)).all()
    sign, logabs = selinv.logdet(prob, lay)
    s2, l2 = np.linalg.slogdet(L @ U)
    assert sign == s2 and abs(logabs - l2) <= 1e-12 * max(1.0, abs(l2))


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_selinv_fixtures(name):
    prob, _, _ = load_fixture(name)
    assert oracle.factor(prob)[0] == 0
    check_against_dense(prob, prob.layers[0])


@pytest.mark.parametrize("values", ["unsym", "mixed"])
@pytest.mark.parametrize("kw", GENERATED, ids=["poisson8", "fem5", "poisson10"])
def test_oracle_selinv_generated(kw, values):
    prob, (rp, ci, v) = poisson_problem(**kw)
    vals = unsym_values(rp, ci, v) if values == "unsym" else mixed_values(rp, ci, v, seed=3)
    prob.fill_layer(0, rp, ci, vals)
    assert oracle.factor(prob)[0] == 0
    check_against_dense(prob, prob.layers[0])


def test_oracle_logdet_sign_indefinite():
    """A matrix with negative pivots: the sign is that of det A (the symmetric permutation leaves it unchanged)."""
    kw = GENERATED[0]
    prob, (rp, ci, v) = poisson_problem(**kw)
    vals = mixed_values(rp, ci, v, seed=4)
    prob.fill_layer(0, rp, ci, vals)
    assert oracle.factor(prob)[0] == 0
    n = prob.n
    A = np.zeros((n, n))
    A[np.repeat(np.arange(n), np.diff(rp)), ci] = vals
    s, la = np.linalg.slogdet(A)
    sign, logabs = selinv.logdet(prob, prob.layers[0])
    assert sign == s and abs(logabs - la) <= 1e-12 * abs(la)
