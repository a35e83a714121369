"""The host side of partial factorization (no GPU): sluh_symbolic_schur keeps the Schur unknowns last, in the caller's order
and in whole supernodes, with a topological supernodal tree; hostlib.schur_order orders any Schur set last; the stored
structure has a slot for every non-zero of L11, U11, L21, U12 and S of a dense partial elimination; and sluh_symbolic
still produces what it produced before the Schur variant existed (digests of its output, taken from that version)."""
import hashlib

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import LUProblem, hostlib
from test_scaled_parity import mixed_values, panel_coords
from test_unsym_skyline_cpu import fill, upwind_matrix


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


# the cases at scale: too large for a dense reference (oracle_partial is theirs); Schur panels of 160 to 1024 rows, so the
# gather walks an L column in several passes, and eliminated supernodes wide enough for the big-tile Schur kernel
def _p16_w256():
    """the 256-column top separator of Poisson 16^3, one Schur supernode"""
    rp, ci, v, perm = _poisson(16, leaf=16)
    return rp, ci, v, _top(rp, perm, 256), perm, dict(relax=32, maxsup=256), False


def _p20_scat():
    """160 random unknowns of Poisson 20^3: Schur destinations shared by updates from every level"""
    rp, ci, v, _ = _poisson(20)
    schur = np.random.default_rng(13).choice(8000, 160, replace=False)
    return rp, ci, v, schur, None, dict(relax=16, maxsup=128), False


def _upwind20():
    (rp, ci, v), perm = upwind_matrix(N=20, frac=0.5, seed=2)
    return rp, ci, v, _top(rp, perm, 400), perm, dict(relax=16, maxsup=128, amalg=0.05), True


def _fem18_w512():
    """the top separator of FEM 18^3 x 3 dof (972 unknowns): Schur supernodes of 512 and 460 columns (double only: the
    doublecomplex path caps supernodes at 256 columns)"""
    rp, ci, v = hostlib.fem3d(18, dof=3)
    perm = hostlib.nd_order(18, dof=3, leaf=32)
    return rp, ci, v, _top(rp, perm, 972), perm, dict(relax=64, maxsup=512), False


def _p32_top():
    """the 1024-unknown top separator of Poisson 32^3 in four 256-column supernodes"""
    rp, ci, v, perm = _poisson(32, leaf=64)
    return rp, ci, v, _top(rp, perm, 1024), perm, dict(relax=32, maxsup=256), False


SCALE_CASES = {"p16_w256": _p16_w256, "p20_scat": _p20_scat, "upwind20": _upwind20, "fem18_w512": _fem18_w512,
               "p32_top": _p32_top}


def case_perm(rp, ci, schur, perm):
    """perm[old] = new with schur[t] -> n - s + t: the geometric ND itself when it already numbers them last, else
    hostlib.schur_order"""
    n, s = len(rp) - 1, len(schur)
    if perm is not None and np.array_equal(perm[schur], np.arange(n - s, n)):
        return np.asarray(perm, np.int32)
    return hostlib.schur_order(rp, ci, schur, leaf=8)


def schur_problem(name, layers=(0,)):
    """-> (LUProblem with nschur, (rowptr, colind, |values|), schur); name from CASES or SCALE_CASES"""
    rp, ci, v, schur, perm, kw, prune = (CASES[name] if name in CASES else SCALE_CASES[name])()
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


def schur_panels(prob, layer, coords=None):
    """S (s, s) read from the Schur panels of layer: every stored entry (r, c) with r, c >= n - s (coords: panel_coords)"""
    n1 = prob.n - prob.nschur
    lrow, lcol, urow, ucol = panel_coords(prob, layer) if coords is None else coords
    S = np.zeros((prob.nschur,) * 2, layer.lval.dtype)
    for r, c, v in ((lrow, lcol, layer.lval), (urow, ucol, layer.uval)):
        m = (r >= n1) & (c >= n1)
        S[r[m] - n1, c[m] - n1] = v[m]
    return S


def oracle_partial(prob, rp, ci, vals):
    """The oracle's partial elimination, a reference that scales: layer 0 filled with vals (float64, or complex128 part by
    part), its eliminated supernodes 0 .. k1 - 1 (columns 0 .. n - s - 1) factored in place by oracle.factor_nodes, which
    leaves S = A22 - A21 A11^-1 A12 in the Schur panels.  -> (info, S (s, s), layer)"""
    fill(prob, rp, ci, vals)
    lay = prob.layers[0]
    k1 = int(np.searchsorted(np.asarray(prob.xsup), prob.n - prob.nschur))
    info, _, _ = oracle.factor_nodes(prob, lay, np.arange(k1))
    return info, schur_panels(prob, lay), lay


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


@pytest.mark.parametrize("complex_", [False, True], ids=["d", "z"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_partial_matches_dense(name, complex_):
    """oracle_partial, the reference of the GPU tests at scale, against the dense A22 - A21 A11^-1 A12 of every small
    case on sign-indefinite values; S is read from the panels, so every entry off the stored pattern is 0 there too"""
    prob, (rp, ci, v), schur = schur_problem(name)
    vals = mixed_values(rp, ci, v, seed=5, complex_=complex_)
    n1 = prob.n - len(schur)
    assert prob.nschur == len(schur)
    info, S, lay = oracle_partial(prob, rp, ci, vals)
    assert info == 0
    assert lay.lval.dtype == (np.complex128 if complex_ else np.float64)
    F = dense_F(rp, ci, vals, np.asarray(prob.perm))
    Sref = F[n1:, n1:] - F[n1:, :n1] @ np.linalg.solve(F[:n1, :n1], F[:n1, n1:])
    assert np.abs(S - Sref).max() <= 1e-13 * np.abs(Sref).max(), np.abs(S - Sref).max() / np.abs(Sref).max()


def _big_tile_sources(prob, n1):
    """eliminated supernodes with m, n >= 96 (updates of the big-tile Schur kernel), from the symbolic structure"""
    ns = np.diff(np.asarray(prob.xsup)).astype(np.int64)
    m = np.asarray(prob.lidx)[np.asarray(prob.lidx_off)[:-1] + 1].astype(np.int64) - ns
    nu = np.asarray(prob.uval_len, np.int64) // np.maximum(ns, 1)
    return int(((m >= 96) & (nu >= 96) & (np.asarray(prob.xsup)[:-1] < n1)).sum())


# (s, widths of the Schur supernodes): every case has eliminated sources for the big-tile kernel and a Schur panel of
# more than 128 rows; the three largest have L columns of more than 512 rows, several passes of the gather's loop
SCALE_SHAPES = {"p16_w256": (256, [256]), "p20_scat": (160, [128, 32]), "upwind20": (400, [128, 128, 128, 16]),
                "fem18_w512": (972, [512, 460]), "p32_top": (1024, [256] * 4)}


@pytest.mark.parametrize("name", sorted(SCALE_CASES))
def test_scale_cases_have_their_shape(name):
    prob, _, schur = schur_problem(name, layers=())
    s, widths = SCALE_SHAPES[name]
    n1 = prob.n - s
    xsup = np.asarray(prob.xsup)
    assert len(schur) == s and n1 in xsup
    assert sorted(np.diff(xsup[xsup >= n1]).tolist(), reverse=True) == widths
    assert _big_tile_sources(prob, n1) > 0
    nsupr = int(prob.lidx[prob.lidx_off[int(np.searchsorted(xsup, n1))] + 1])     # rows of the first Schur L panel
    assert nsupr == s and (nsupr > 512) == (s > 512)


def test_fill_layer_refuses_complex():
    """the host fill writes doubles: complex values, or a complex128 layer, would be silently corrupted"""
    prob, (rp, ci, v), _ = schur_problem("p8_top")
    vals = mixed_values(rp, ci, v, seed=5, complex_=True)
    before = prob.layers[0].lval.copy()
    with pytest.raises(TypeError, match="part by part"):
        prob.fill_layer(0, rp, ci, vals)
    assert np.array_equal(prob.layers[0].lval, before)
    prob.dtype = np.dtype(np.complex128)
    prob.add_layer(0)
    with pytest.raises(TypeError, match="part by part"):
        prob.fill_layer(0, rp, ci, vals.real)
    # the part-by-part fill gives the values of each part exactly
    fill(prob, rp, ci, vals)
    re, im = schur_problem("p8_top")[0], schur_problem("p8_top")[0]
    re.fill_layer(0, rp, ci, vals.real)
    im.fill_layer(0, rp, ci, vals.imag)
    assert np.array_equal(prob.layers[0].lval, re.layers[0].lval + 1j * im.layers[0].lval)
    assert np.array_equal(prob.layers[0].uval, re.layers[0].uval + 1j * im.layers[0].uval)
