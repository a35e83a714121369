"""The host side of partial factorization (no GPU): sluh_symbolic_schur keeps the Schur unknowns last, in the caller's order
and in whole supernodes, with a topological supernodal tree; hostlib.schur_order orders any Schur set last; the stored
structure has a slot for every non-zero of L11, U11, L21, U12 and S of a dense partial elimination; and sluh_symbolic
still produces what it produced before the Schur variant existed (digests of its output, taken from that version)."""
import hashlib

import numpy as np
import pytest

from superlu_dist_b200 import LUProblem, hostlib
from test_scaled_parity import mixed_values, panel_coords
from test_unsym_skyline_cpu import upwind_matrix


# ------------------------------------------------------------------------------------------------------------ the cases
def _poisson(N, leaf=4):
    rp, ci, v = hostlib.poisson3d(N)
    return rp, ci, v, hostlib.nd_order(N, leaf=leaf)


def _top(rp, perm, s):
    """the last s unknowns of perm (for the geometric ND: the top-level separator), in perm's order"""
    return np.argsort(perm)[len(rp) - 1 - s:]


def _p8_top():
    rp, ci, v, perm = _poisson(8)
    return rp, ci, v, _top(rp, perm, 64), perm, dict(relax=8, maxsup=32), False


def _p8_scattered():
    rp, ci, v, _ = _poisson(8)
    schur = np.random.default_rng(11).choice(512, 40, replace=False)
    return rp, ci, v, schur, None, dict(relax=8, maxsup=32), False


def _fem5_nodes():
    rp, ci, v = hostlib.fem3d(5, dof=3)
    nodes = np.random.default_rng(12).choice(125, 12, replace=False)
    schur = (3 * nodes[:, None] + np.arange(3)).ravel()          # every dof of a node
    return rp, ci, v, schur, None, dict(relax=8, maxsup=64), False


def _p8_one():
    rp, ci, v, _ = _poisson(8)
    return rp, ci, v, np.array([137]), None, dict(relax=8, maxsup=32), False


def _p8_wide():
    rp, ci, v, perm = _poisson(8)
    return rp, ci, v, _top(rp, perm, 64), perm, dict(relax=8, maxsup=16), False


def _p8_two():
    """two disjoint interfaces: the planes x = 2 and x = 5"""
    rp, ci, v, _ = _poisson(8)
    x = np.arange(512) % 8
    return rp, ci, v, np.nonzero((x == 2) | (x == 5))[0], None, dict(relax=8, maxsup=32), False


def _upwind_small():
    (rp, ci, v), perm = upwind_matrix(N=10, frac=0.5, seed=2)
    return rp, ci, v, _top(rp, perm, 100), perm, dict(relax=8, maxsup=64, amalg=0.05), True


CASES = {"p8_top": _p8_top, "p8_scattered": _p8_scattered, "fem5_nodes": _fem5_nodes, "p8_one": _p8_one,
         "p8_wide": _p8_wide, "p8_two": _p8_two, "upwind_small": _upwind_small}


def case_perm(rp, ci, schur, perm):
    """perm[old] = new with schur[t] -> n - s + t: the geometric ND itself when it already numbers them last, else
    hostlib.schur_order"""
    n, s = len(rp) - 1, len(schur)
    if perm is not None and np.array_equal(perm[schur], np.arange(n - s, n)):
        return np.asarray(perm, np.int32)
    return hostlib.schur_order(rp, ci, schur, leaf=8)


def schur_problem(name, layers=(0,)):
    """-> (LUProblem with nschur, (rowptr, colind, |values|), schur)"""
    rp, ci, v, schur, perm, kw, prune = CASES[name]()
    perm = case_perm(rp, ci, schur, perm)
    prob = LUProblem.from_matrix(rp, ci, v, perm, layers=() if prune else layers, nschur=len(schur), **kw)
    if prune:
        prob.prune_u(rp, ci)
        for z in layers:
            prob.add_layer(z)
            prob.fill_layer(z, rp, ci, v)
    return prob, (rp, ci, v), schur


def dense_F(rp, ci, vals, perm):
    n = len(rp) - 1
    F = np.zeros((n, n), np.asarray(vals).dtype)
    rows = np.repeat(np.arange(n), np.diff(rp))
    F[perm[rows], perm[ci]] = vals
    return F


def partial_eliminate(F, n1):
    """unpivoted elimination of the first n1 columns: L21 / L11 strictly below the diagonal, U11 / U12 on and above it,
    S = A22 - A21 A11^-1 A12 in the trailing block"""
    W = F.copy()
    for k in range(n1):
        W[k + 1:, k] /= W[k, k]
        W[k + 1:, k + 1:] -= np.outer(W[k + 1:, k], W[k, k + 1:])
    return W


# ------------------------------------------------------------------------------------------------------------ the tests
def _digest(sym):
    h = hashlib.sha256()
    for a in (sym.perm, sym.xsup, sym.setree, sym.lidx_off, sym.lidx, sym.uidx_off, sym.uidx, sym.lval_off, sym.uval_off,
              np.array([sym.ops_fact, sym.ops_schur])):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:32]


# digests of sluh_symbolic's output before sluh_symbolic_schur existed
DIGESTS = {
    "p12": ("poisson", 12, 1, 8, 8, 32, 0.05, "b0f5ddd99922733730c1ebff99c20aa4"),
    "p16": ("poisson", 16, 1, 16, 32, 256, 0.05, "6c124562da3c2ba1e83fdac6e6c3629e"),
    "fem6": ("fem", 6, 3, 8, 16, 128, 0.0, "ce17cf2e24213674b3003f3ca853f4b3"),
    "p9_noperm": ("poisson", 9, 1, 0, 8, 64, 0.3, "e1a84760a1546bc14d18c991e3db42a7"),
}


@pytest.mark.parametrize("name", sorted(DIGESTS))
def test_symbolic_unchanged(name):
    family, N, dof, leaf, relax, maxsup, amalg, want = DIGESTS[name]
    rp, ci, _ = hostlib.poisson3d(N) if family == "poisson" else hostlib.fem3d(N, dof=dof)
    perm = None if leaf == 0 else hostlib.nd_order(N, dof=dof, leaf=leaf)
    n = len(rp) - 1
    assert _digest(hostlib.Symbolic(n, rp, ci, perm, relax, maxsup, amalg)) == want
    assert _digest(hostlib.Symbolic(n, rp, ci, perm, relax, maxsup, amalg, nschur=0)) == want


@pytest.mark.parametrize("name", sorted(CASES))
def test_schur_last_and_whole_supernodes(name):
    prob, (rp, ci, v), schur = schur_problem(name, layers=())
    n, s = prob.n, len(schur)
    perm, xsup = np.asarray(prob.perm), np.asarray(prob.xsup)
    assert np.array_equal(perm[schur], np.arange(n - s, n))
    assert n - s in xsup
    widths = np.diff(xsup)
    maxsup = CASES[name]()[5]["maxsup"]
    assert widths.max() <= maxsup
    assert (xsup >= n - s).sum() - 1 >= -(-s // maxsup)      # Schur supernodes
    st = np.asarray(prob.setree)
    k = np.arange(prob.nsupers)
    assert np.all((st > k) | (st == prob.nsupers))


@pytest.mark.parametrize("name", sorted(CASES))
def test_structure_holds_partial_elimination(name):
    prob, (rp, ci, v), schur = schur_problem(name)
    n, s = prob.n, len(schur)
    F = dense_F(rp, ci, mixed_values(rp, ci, v, seed=5), np.asarray(prob.perm))
    W = partial_eliminate(F, n - s)
    lrow, lcol, urow, ucol = panel_coords(prob, prob.layers[0])
    u = urow >= 0
    stored = np.zeros((n, n), bool)
    stored[np.concatenate([lrow, urow[u]]), np.concatenate([lcol, ucol[u]])] = True
    missing = (W != 0) & ~stored
    assert not missing.any(), np.argwhere(missing)[:5]


def test_schur_order_rejects_bad_sets():
    rp, ci, _ = hostlib.poisson3d(4)
    with pytest.raises(ValueError):
        hostlib.schur_order(rp, ci, [1, 1])
    with pytest.raises(ValueError):
        hostlib.schur_order(rp, ci, [64])
    with pytest.raises(ValueError):
        hostlib.Symbolic(64, rp, ci, None, nschur=65)
