"""Partial factorization at scale (slu_b200_schur_* and the z twins) against the oracle's partial elimination
(test_schur_symbolic_cpu.oracle_partial) on SCALE_CASES: Schur panels of 160 to 1024 rows, so the gather copies an L
column in several passes; 256- and 512-column eliminated supernodes whose updates take the big-tile DMMA Schur kernel into
destinations that are never factored, with look-ahead on and off; Schur destinations shared by every level.

S is checked against the oracle entry by entry (and exactly 0 off the stored pattern), also on row- and column-scaled
matrices, where a normwise bar would hide wrong rows of small scale; the eliminated panels against the oracle's; the
composed solve condense -> S -> expand against the whole sparse system; and a zero pivot in the middle of a wide
eliminated supernode."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from superlu_dist_b200 import capi
from test_gpu_schur import TOL, stored_mask
from test_scaled_parity import exponents, ldexp, mixed_values, permuted, scaled
from test_schur_symbolic_cpu import SCALE_CASES, oracle_partial, schur_panels, schur_problem

pytestmark = pytest.mark.gpu
# doublecomplex supernodes are at most 256 columns wide: fem18_w512 is double only
PRECISIONS = [pytest.param(name, dt, id=f"{name}-{dt}") for name in sorted(SCALE_CASES) for dt in ("d", "z")
              if not (name == "fem18_w512" and dt == "z")]


@functools.lru_cache(maxsize=None)
def reference(name, dt):
    """-> (problem, (rowptr, colind, values), S, eliminated L values, eliminated U values) of the oracle's partial
    elimination of the sign-indefinite matrix of case `name`; dt 'z': complex values"""
    prob, (rp, ci, v), _ = schur_problem(name)
    vals = mixed_values(rp, ci, v, seed=7, complex_=dt == "z")
    info, S, lay = oracle_partial(prob, rp, ci, vals)
    assert info == 0
    k1 = first_schur(prob)
    return prob, (rp, ci, vals), S, lay.lval[:lay.lval_off[k1]].copy(), lay.uval[:lay.uval_off[k1]].copy()


def first_schur(prob):
    return int(np.searchsorted(np.asarray(prob.xsup), prob.n - prob.nschur))


def handle(prob, **opt):
    """a Schur handle on a fresh layer 0 (the oracle's layer stays as it is)"""
    prob.add_layer(0)
    return capi.SchurHandle(prob, prob.nschur, **opt)


def factored(name, dt, vals=None, **opt):
    prob, (rp, ci, v), _, _, _ = reference(name, dt)
    h = handle(prob, **opt)
    h.fill_csr(rp, ci, v if vals is None else vals, prob.perm)
    assert h.factor() == 0
    return h


def check_s(S, Sref, tol=TOL):
    err = np.abs(S - Sref).max() / np.abs(Sref).max()
    assert err <= tol, err


@pytest.mark.parametrize("name,dt", PRECISIONS)
def test_schur_and_eliminated_panels_match_oracle(name, dt):
    prob, _, Sref, lref, uref = reference(name, dt)
    h = factored(name, dt)
    S = h.schur()
    check_s(S, Sref)
    n1 = prob.n - prob.nschur
    assert np.all(S[~stored_mask(prob, n1)] == 0)
    assert S.tobytes() == h.schur().tobytes()                                # bit-identical
    h.download()
    lay = prob.layers[0]
    k1 = first_schur(prob)
    for got, want in ((lay.lval[:lay.lval_off[k1]], lref), (lay.uval[:lay.uval_off[k1]], uref)):
        assert np.abs(got - want).max() <= TOL * np.abs(want).max(), np.abs(got - want).max() / np.abs(want).max()
    # the downloaded Schur panels are S, bit for bit
    assert np.array_equal(schur_panels(prob, lay), S)
    h.close()


@pytest.mark.parametrize("dt", ["d", "z"])
@pytest.mark.parametrize("name", ["p20_scat", "p32_top"])
def test_lookahead_on_and_off(name, dt):
    """the look-ahead's urgent / bulk split over two streams and the single-stream level loop give the same S"""
    h0, h1 = factored(name, dt), factored(name, dt, no_lookahead=1)
    S0, S1 = h0.schur(), h1.schur()
    check_s(S1, S0, 1e-12)
    h0.close()
    h1.close()


@pytest.mark.parametrize("name,dt", [("p32_top", "d"), ("upwind20", "d"), ("p16_w256", "z")])
def test_scaled_matrix_gives_scaled_schur(name, dt):
    """A' = 2^er A 2^ec (|er|, |ec| <= 20) has S' = 2^er2 S 2^ec2 over the Schur rows and columns: S' un-scaled meets the
    bar against the oracle's S of the unscaled matrix entry by entry in each entry's own scale"""
    prob, (rp, ci, vals), Sref, _, _ = reference(name, dt)
    er, ec = exponents(prob.n, 20, seed=3)
    n1 = prob.n - prob.nschur
    er2, ec2 = permuted(prob, er)[n1:], permuted(prob, ec)[n1:]
    assert er2.max() - er2.min() >= 30
    h = factored(name, dt, vals=scaled(rp, ci, vals, er, ec))
    S = ldexp(h.schur(), -(er2[:, None] + ec2[None, :]))
    check_s(S, Sref)
    h.close()


@pytest.mark.parametrize("name,dt", PRECISIONS)
def test_composed_solve(name, dt):
    """condense, a dense solve with S, expand: the solution of the whole sparse system F x = b"""
    prob, (rp, ci, vals), _, _, _ = reference(name, dt)
    n, n1 = prob.n, prob.n - prob.nschur
    perm = np.asarray(prob.perm)
    rows = np.repeat(np.arange(n), np.diff(rp))
    F = sp.csr_matrix((vals, (perm[rows], perm[ci])), shape=(n, n))
    fnorm = abs(F).sum(axis=1).max()
    h = factored(name, dt)
    S = h.schur()
    rng = np.random.default_rng(4)
    for nrhs in (1, 17):
        b = rng.standard_normal((nrhs, n))
        if dt == "z":
            b = b + 1j * rng.standard_normal((nrhs, n))
        y = h.condense(b[0] if nrhs == 1 else b).reshape(nrhs, n)
        y[:, n1:] = np.linalg.solve(S, y[:, n1:].T).T
        x = h.expand(y[0] if nrhs == 1 else y).reshape(nrhs, n)
        for j in range(nrhs):
            res = np.linalg.norm(F @ x[j] - b[j]) / (fnorm * np.linalg.norm(x[j]) + np.linalg.norm(b[j]))
            assert res <= 1e-12, (nrhs, j, res)
        if name in ("p20_scat", "upwind20"):
            xs = spla.spsolve(F.tocsc(), b.T).reshape(n, nrhs).T
            assert np.abs(x - xs).max() <= TOL * np.abs(xs).max()
    h.close()


@pytest.mark.parametrize("dt", ["d", "z"])
def test_zero_pivot_in_wide_eliminated_supernode(dt):
    """one column of A11 zero, in the middle of a 256-column eliminated supernode: factor reports the oracle's info, and
    the same handle refilled with good values gives the oracle's S"""
    name = "p32_top"
    prob, (rp, ci, vals), Sref, _, _ = reference(name, dt)
    xsup = np.asarray(prob.xsup)
    n1 = prob.n - prob.nschur
    wide = np.nonzero((np.diff(xsup) == 256) & (xsup[:-1] < n1))[0]
    assert len(wide)
    j = int(xsup[wide[0]] + 128)
    perm = np.asarray(prob.perm)
    rows = np.repeat(np.arange(prob.n), np.diff(rp))
    bad = np.where((perm[ci] == j) & (perm[rows] < n1), 0, vals).astype(vals.dtype)
    assert (bad != vals).sum() >= 3
    prob.add_layer(0)
    info_ref, _, _ = oracle_partial(prob, rp, ci, bad)
    assert info_ref == j + 1
    h = handle(prob)
    h.fill_csr(rp, ci, bad, prob.perm)
    assert h.factor() == info_ref
    with pytest.raises(RuntimeError, match="needs a successful"):
        h.schur()
    h.fill_csr(rp, ci, vals, prob.perm)
    assert h.factor() == 0
    check_s(h.schur(), Sref)
    h.close()
