"""oracle/selinv.py on doublecomplex layers, the reference for slu_b200_z_selinv: H = F^-T (a plain transpose, not the
conjugate) at every stored position of L + U against a dense inverse of the oracle's own factors, on the complex golden
fixture, on complex problems of the generated shapes, and on a complex-symmetric shifted matrix; and the complex
log-determinant (log |det|, phase exp(i theta)) against numpy.linalg.slogdet."""
import numpy as np
import pytest

from oracle import oracle, selinv
from test_scaled_parity import make_problem, mixed_values, panel_coords
from util import complex_problem, load_fixture, poisson_problem

TOL = 1e-10
GENERATED = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=5, leaf=4, relax=8, maxsup=200, fem=3),
             dict(N=10, leaf=8, relax=16, maxsup=128)]
TWO_PI = 2.0 * np.pi


def complex_logdet(prob, lay):
    """(sign, log |det F|) of a complex layer from its pivots: sum of log |u_ii|, sign = exp(i theta) with theta the sum of
    arg u_ii reduced modulo 2 pi (the phase slu_b200_z_logdet returns)"""
    xsup = np.asarray(prob.xsup, np.int64)
    logabs, theta = 0.0, 0.0
    for k in np.nonzero(lay.held)[0]:
        ns = int(xsup[k + 1] - xsup[k])
        nsupr = int(prob.lidx[prob.lidx_off[k] + 1])
        o = int(lay.lval_off[k])
        d = lay.lval[o:o + ns * nsupr].reshape(ns, nsupr)[np.arange(ns), np.arange(ns)]
        logabs += float(np.sum(np.log(np.abs(d))))
        theta += float(np.sum(np.angle(d)))
    return np.exp(1j * np.remainder(theta, TWO_PI)), logabs


def shifted_values(rp, ci, v, eta=0.5):
    """K - (E + i eta) I on the pattern of the real symmetric K (hostlib.poisson3d): complex symmetric, not Hermitian.  E = trace(K) / n lies
    inside K's spectrum; Im A = -eta I is definite, so every leading principal block is nonsingular (unpivoted LU exists)."""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    dg = rows == np.asarray(ci)
    v = np.asarray(v, np.float64)
    E = v[dg].mean()
    return np.where(dg, v - (E + 1j * eta), v + 0j)


def shifted_problem(kw, eta=0.5):
    """(problem holding K - (E + i eta) I, rp, ci, values)"""
    _, (rp, ci, v) = poisson_problem(**kw)
    vals = shifted_values(rp, ci, v, eta)
    return make_problem(kw, vals), rp, ci, vals


def check_against_dense(prob, lay):
    L, U = prob.dense(lay, True)
    F = L @ U
    G = np.linalg.inv(F)
    hl, hu = selinv.selinv(prob, lay)
    assert hl.dtype == np.complex128 and hu.dtype == np.complex128
    lrow, lcol, urow, ucol = panel_coords(prob, lay)
    scale = np.abs(G).max()
    assert np.abs(hl - G.T[lrow, lcol]).max() <= TOL * scale
    u = urow >= 0
    assert np.abs(hu[u] - G.T[urow[u], ucol[u]]).max(initial=0.0) <= TOL * scale
    dg = lrow == lcol
    d = G[lrow[dg], lcol[dg]]
    assert dg.sum() == prob.n and (np.abs(hl[dg] - d) <= TOL * np.abs(d)).all()
    sign, logabs = complex_logdet(prob, lay)
    s2, l2 = np.linalg.slogdet(F)
    assert abs(sign - s2) <= 1e-12 and abs(logabs - l2) <= 1e-12 * max(1.0, abs(l2))
    return G


def test_oracle_selinv_complex_fixture():
    prob, _, _ = load_fixture("cg20_pzdrive3d")
    assert prob.dtype == np.complex128
    assert oracle.factor(prob)[0] == 0
    check_against_dense(prob, prob.layers[0])


@pytest.mark.parametrize("kw", GENERATED, ids=["poisson8", "fem5", "poisson10"])
def test_oracle_selinv_complex_generated(kw):
    prob = complex_problem(**kw)
    assert oracle.factor(prob)[0] == 0
    check_against_dense(prob, prob.layers[0])


@pytest.mark.parametrize("kw", GENERATED[::2], ids=["poisson8", "poisson10"])
def test_oracle_selinv_complex_symmetric_shift(kw):
    """A = K - (E + i eta) I: A^-1 is complex symmetric, and the transpose (not the conjugate) reproduces it."""
    prob, rp, ci, vals = shifted_problem(kw)
    assert oracle.factor(prob)[0] == 0
    G = check_against_dense(prob, prob.layers[0])
    assert np.abs(G - G.T).max() <= TOL * np.abs(G).max()
    assert np.abs(G - G.conj().T).max() > 1e-3 * np.abs(G).max()


def test_complex_logdet_matches_slogdet_of_a():
    """The phase of det A from the pivots of F = P A P^T (the symmetric permutation leaves det unchanged), on values whose
    diagonal carries random unit phases, so that theta wraps around 2 pi many times."""
    kw = GENERATED[2]
    _, (rp, ci, v) = poisson_problem(**kw)
    vals = mixed_values(rp, ci, v, seed=7, complex_=True)
    prob = make_problem(kw, vals)
    n = prob.n
    A = np.zeros((n, n), np.complex128)
    A[np.repeat(np.arange(n), np.diff(rp)), ci] = vals
    assert oracle.factor(prob)[0] == 0
    sign, logabs = complex_logdet(prob, prob.layers[0])
    s2, l2 = np.linalg.slogdet(A)
    assert abs(abs(sign) - 1.0) <= 1e-15
    assert abs(sign - s2) <= 1e-12 and abs(logabs - l2) <= 1e-12 * abs(l2)
