"""Scale-exact parity: every factorization route on sign-indefinite matrices whose rows and columns are scaled by powers
of two spanning up to 2^(+-20), compared with the oracle entry by entry in each entry's own scale.

The generated problems of the other tests are M-matrices of uniform O(1) scale: nothing cancels (L U = |L| |U|), and a
normwise bar (max |a - b| / max |b| over an arena) lets whole rows of small entries be wrong.  Here the values are
random-sign and strictly row-diagonally dominant (an unpivoted LU exists, growth <= 2), and A' = 2^er A 2^ec is exact.
Its factors are L' = D_r L D_r^-1 and U' = D_r U D_c (D = diag(2^e) in the factored ordering), so multiplying them back
by 2^(er_k - er_i) (strict lower L) and 2^(-er_i - ec_j) (U) gives the factors of A, bit for bit when the arithmetic is
FP64 throughout: multiplies, FMAs, reciprocals and sums all commute with power-of-two scaling.  The bar of the other
parity tests (rel_err < 1e-10) then holds for every entry relative to the largest entry of its own scale class.

The int8 tensor-core path (slu_ozaki.cu) is not equivariant: its slices are scaled per row of the L operand and per
column of the U operand, which absorb neither 2^er_k, so its error grows as (max r / min r)^2 (DESIGN 4b).  It is
tested here at E = 0 only (cancellation through the slices); by default it is off."""
import functools

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi
from superlu_dist_b200.problem import BC_HEADER, BR_HEADER, LB_DESCRIPTOR, UB_DESCRIPTOR
from util import load_fixture, poisson_problem, rel_err

TOL = 1e-10


# ---------------------------------------------------------------------------------------------------------- the harness
def mixed_values(rp, ci, v, seed, complex_=False):
    """Non-symmetric, sign-indefinite values on the pattern of (rp, ci): every off-diagonal entry |v| U(0.5, 1.5) with a
    random sign, every diagonal entry (the row's off-diagonal 1-norm + 1) with a random sign -- strictly row-diagonally
    dominant.  complex_: random-sign real and imaginary parts off the diagonal (each |v| U(0.5, 1.5)), on the diagonal
    (the row's 1-norm of moduli + 1) times a random unit phase."""
    rng = np.random.default_rng(seed)
    n, nnz = len(rp) - 1, len(ci)
    rows = np.repeat(np.arange(n), np.diff(rp))
    off = rows != np.asarray(ci)
    mag = np.abs(np.asarray(v, np.float64))

    def part():
        return mag * rng.uniform(0.5, 1.5, nnz) * rng.choice([-1.0, 1.0], nnz)

    if not complex_:
        w = np.where(off, part(), 0.0)
        d = (np.bincount(rows, np.abs(w), n) + 1.0) * rng.choice([-1.0, 1.0], n)
        return np.where(off, w, d[rows])
    w = np.where(off, part() + 1j * part(), 0.0)
    d = (np.bincount(rows, np.abs(w), n) + 1.0) * np.exp(1j * rng.uniform(0.0, 2 * np.pi, n))
    return np.where(off, w, d[rows])


def exponents(n, E, seed):
    """Integer row and column exponents, uniform in [-E, E] (original ordering)."""
    rng = np.random.default_rng(10_000 + seed)
    return rng.integers(-E, E + 1, n), rng.integers(-E, E + 1, n)


def ldexp(x, e):
    """x * 2^e exactly (real or complex)."""
    if np.iscomplexobj(x):
        return np.ldexp(x.real, e) + 1j * np.ldexp(x.imag, e)
    return np.ldexp(x, e)


def scaled(rp, ci, vals, er, ec):
    """A' = 2^er A 2^ec on the CSR values."""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    return ldexp(vals, er[rows] + ec[np.asarray(ci)])


def permuted(prob, e):
    """Exponents of the original ordering -> the factored ordering (perm[old] = new)."""
    out = np.empty_like(e)
    out[np.asarray(prob.perm)] = e
    return out


def panel_coords(prob, layer):
    """(row, col) in the factored ordering of every stored value of layer.lval and layer.uval -> (lrow, lcol, urow,
    ucol); -1 where the layer holds nothing.  The walk of LUProblem.dense, vectorised per block: L panel k is column-
    major ns x nsupr over the rows of its blocks; U panel k is, per block column jb and column c of it, the skyline
    segment of rows fst .. klst - 1 (zero-padded segments included)."""
    lrow = np.full(len(layer.lval), -1, np.int64)
    lcol = np.full(len(layer.lval), -1, np.int64)
    urow = np.full(len(layer.uval), -1, np.int64)
    ucol = np.full(len(layer.uval), -1, np.int64)
    xsup = np.asarray(prob.xsup, np.int64)
    for k in np.nonzero(layer.held)[0]:
        f, klst = int(xsup[k]), int(xsup[k + 1])
        ns = klst - f
        if prob.lidx_off[k + 1] > prob.lidx_off[k]:
            idx = prob.lidx[prob.lidx_off[k]:prob.lidx_off[k + 1]]
            nsupr, w, rows = int(idx[1]), BC_HEADER, []
            for _ in range(int(idx[0])):
                nb = int(idx[w + 1])
                rows.append(idx[w + LB_DESCRIPTOR:w + LB_DESCRIPTOR + nb])
                w += LB_DESCRIPTOR + nb
            rows = np.concatenate(rows).astype(np.int64)
            assert len(rows) == nsupr, k
            o = int(layer.lval_off[k])
            assert int(layer.lval_off[k + 1]) - o == ns * nsupr, k
            lrow[o:o + ns * nsupr] = np.tile(rows, ns)
            lcol[o:o + ns * nsupr] = np.repeat(np.arange(f, klst), nsupr)
        if prob.uidx_off[k + 1] > prob.uidx_off[k]:
            idx = prob.uidx[prob.uidx_off[k]:prob.uidx_off[k + 1]]
            o, u = int(layer.uval_off[k]), BR_HEADER
            for _ in range(int(idx[0])):
                jb = int(idx[u])
                jf, jns = int(xsup[jb]), int(xsup[jb + 1] - xsup[jb])
                fst = idx[u + UB_DESCRIPTOR:u + UB_DESCRIPTOR + jns].astype(np.int64)
                seg = np.maximum(klst - fst, 0)
                tot = int(seg.sum())
                start = np.repeat(np.cumsum(seg) - seg, seg)
                urow[o:o + tot] = np.repeat(fst, seg) + (np.arange(tot) - start)
                ucol[o:o + tot] = np.repeat(np.arange(jf, jf + jns), seg)
                o += tot
                u += UB_DESCRIPTOR + jns
            assert o == int(layer.uval_off[k + 1]), k
    return lrow, lcol, urow, ucol


def unscale(prob, layer, er_p, ec_p, coords=None):
    """Factors of A' -> factors of A, exactly: the strict lower part of L times 2^(er_k - er_i), U (with the diagonal
    blocks stored in the L panels) times 2^(-er_i - ec_j).  er_p, ec_p: exponents in the factored ordering.
    -> (lval, uval) new arrays."""
    lrow, lcol, urow, ucol = panel_coords(prob, layer) if coords is None else coords
    held_l, held_u = lrow >= 0, urow >= 0
    r, c = np.where(held_l, lrow, 0), np.where(held_l, lcol, 0)
    el = np.where(r > c, er_p[c] - er_p[r], -er_p[r] - ec_p[c])
    r, c = np.where(held_u, urow, 0), np.where(held_u, ucol, 0)
    eu = -er_p[r] - ec_p[c]
    return ldexp(layer.lval, np.where(held_l, el, 0)), ldexp(layer.uval, np.where(held_u, eu, 0))


def make_problem(kw, vals):
    """A fresh problem on the structure of poisson_problem(**kw) holding `vals` (float64 or complex128; LUProblem.
    fill_layer takes float64, so a complex matrix is filled part by part, as util.complex_problem does)."""
    prob, (rp, ci, _) = poisson_problem(**kw)
    if not np.iscomplexobj(vals):
        prob.fill_layer(0, rp, ci, vals)
        return prob
    lay = prob.layers[0]
    prob.fill_layer(0, rp, ci, vals.real)
    lre, ure = lay.lval.copy(), lay.uval.copy()
    prob.fill_layer(0, rp, ci, vals.imag)
    prob.dtype = np.dtype(np.complex128)
    lay.lval, lay.uval = lre + 1j * lay.lval, ure + 1j * lay.uval
    return prob


def pattern(kw):
    _, (rp, ci, v) = poisson_problem(**kw)
    return rp, ci, v


# -------------------------------------------------------------------------------------------------------- CPU: the harness
def test_panel_coords_match_dense_walk():
    """panel_coords places every stored value where LUProblem.dense does: on a generated problem and on the reference's
    unsym360_mmd dump, whose packed U columns are zero-padded above their first nonzero."""
    probs = [load_fixture("unsym360_mmd")[0], make_problem(dict(N=6, leaf=4, relax=8, maxsup=32),
                                                           mixed_values(*pattern(dict(N=6, leaf=4, relax=8, maxsup=32)), 3))]
    for prob in probs:
        lay = prob.layers[0]
        L, U = prob.dense(lay, factored=True)
        lrow, lcol, urow, ucol = panel_coords(prob, lay)
        assert (lrow >= 0).all() and (urow >= 0).all()
        low = lrow > lcol
        assert np.array_equal(L[lrow[low], lcol[low]], lay.lval[low])
        assert np.array_equal(U[lrow[~low], lcol[~low]], lay.lval[~low])
        assert np.array_equal(U[urow, ucol], lay.uval)
        assert (urow < ucol).all()                                  # U panels hold only the strict upper part
        # no position is stored twice
        n = prob.n
        keys = np.concatenate([lrow * n + lcol, urow * n + ucol])
        assert len(np.unique(keys)) == len(keys)


@pytest.mark.parametrize("kw,complex_", [(dict(N=10, leaf=8, relax=8, maxsup=32), False),
                                         (dict(N=6, leaf=4, relax=8, maxsup=200, fem=3), False),
                                         (dict(N=8, leaf=4, relax=8, maxsup=32), True)],
                         ids=["poisson10", "fem6", "poisson8_complex"])
def test_oracle_is_scale_exact(kw, complex_):
    """The oracle on A' = 2^er A 2^ec (E = 20), unscaled, is bit for bit the oracle on A: pins the harness."""
    rp, ci, v = pattern(kw)
    vals = mixed_values(rp, ci, v, seed=5, complex_=complex_)
    ref = make_problem(kw, vals)
    assert oracle.factor(ref)[0] == 0
    er, ec = exponents(len(rp) - 1, 20, seed=5)
    assert er.min() < -15 and er.max() > 15
    prob = make_problem(kw, scaled(rp, ci, vals, er, ec))
    assert oracle.factor(prob)[0] == 0
    lval, uval = unscale(prob, prob.layers[0], permuted(prob, er), permuted(prob, ec))
    assert np.array_equal(lval, ref.layers[0].lval) and np.array_equal(uval, ref.layers[0].uval)
    # the scaling is not trivial: the factors of A' differ from those of A by orders of magnitude
    assert rel_err(prob.layers[0].lval, ref.layers[0].lval) > 1.0


def test_mixed_values_are_sign_indefinite_and_dominant():
    rp, ci, v = pattern(dict(N=6, fem=3, maxsup=200))
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    for complex_ in (False, True):
        a = mixed_values(rp, ci, v, seed=1, complex_=complex_)
        off = rows != ci
        d = np.abs(a[~off])
        assert np.all(d > np.bincount(rows[off], np.abs(a[off]), len(rp) - 1))
        parts = [a.real, a.imag] if complex_ else [a]
        for p in parts:
            assert (p[off] > 0).any() and (p[off] < 0).any()
        if not complex_:
            assert (a[~off] > 0).any() and (a[~off] < 0).any()


# ------------------------------------------------------------------------------------------------------------ GPU routes
_SMALL = dict(N=10, leaf=8, relax=8, maxsup=32)
_FEM6 = dict(N=6, leaf=4, relax=8, maxsup=200, fem=3)
_W256 = dict(N=16, leaf=16, relax=32, maxsup=256)           # a 256-column top separator
_W512 = dict(N=18, leaf=32, relax=64, maxsup=512, fem=3)    # supernodes of 486 and 512 columns
_NARROW = dict(N=24, leaf=8, relax=8, maxsup=8)             # 64-column tiles span 8 or more destination panels
_MANY = dict(N=20, leaf=32, relax=64, maxsup=256, fem=3)    # many waves of 128 x 64 tiles
_W2 = dict(N=24, leaf=32, relax=64, maxsup=512)             # 576-column top separator -> 512 + 64
_K2 = dict(N=18, leaf=16, relax=32, maxsup=256)
_K4 = dict(N=20, leaf=32, relax=64, maxsup=400)
_Z128 = dict(N=12, leaf=8, relax=16, maxsup=128)
_Z200 = dict(N=5, leaf=4, relax=8, maxsup=200, fem=3)
_PROBLEMS = dict(small=_SMALL, fem6=_FEM6, w256=_W256, w512=_W512, narrow=_NARROW, many=_MANY, w2=_W2, k2=_K2, k4=_K4,
                 z128=_Z128, z200=_Z200)
_NAMES = {id(kw): name for name, kw in _PROBLEMS.items()}


@functools.lru_cache(maxsize=2)
def _reference(name, seed, complex_):
    """The oracle's factors of the unscaled mixed-sign matrix -> (lval, uval)."""
    kw = _PROBLEMS[name]
    rp, ci, v = pattern(kw)
    ref = make_problem(kw, mixed_values(rp, ci, v, seed, complex_))
    assert oracle.factor(ref)[0] == 0
    return ref.layers[0].lval, ref.layers[0].uval


def _widest(prob):
    return int(np.diff(np.asarray(prob.xsup)).max())


def _big_tiles(prob):
    """Updates with m, n >= 96 (the schur_kernel_h tiles), from the symbolic structure."""
    ns = np.diff(np.asarray(prob.xsup)).astype(np.int64)
    m = np.asarray(prob.lidx)[np.asarray(prob.lidx_off)[:-1] + 1].astype(np.int64) - ns
    n = np.asarray(prob.uval_len, dtype=np.int64) // np.maximum(ns, 1)
    return int(((m >= 96) & (n >= 96)).sum())


def _fp64(st):
    assert st.reserved[1] == 0 and int(st.reserved[3]) == 0     # no update took the int8 slices


def _int8(slices):
    def check(st):
        assert st.reserved[1] > 0 and int(st.reserved[3]) == slices
    return check


def _factor_scaled(kw, E, seed=0, complex_=False, **opt):
    """Factor A' on the GPU -> (info, stats, problem, unscaled (lval, uval))."""
    rp, ci, v = pattern(kw)
    vals = mixed_values(rp, ci, v, seed, complex_)
    er, ec = exponents(len(rp) - 1, E, seed)
    prob = make_problem(kw, scaled(rp, ci, vals, er, ec))
    info, st = (capi.pzgstrf3d if complex_ else capi.pdgstrf3d)(prob, 0, **opt)
    return info, st, prob, unscale(prob, prob.layers[0], permuted(prob, er), permuted(prob, ec))


# (route id, problem, options, route check, structural check)
ROUTES = [
    ("dmma_small", _SMALL, dict(tc_slices=-1), _fp64, lambda p: _widest(p) <= 32),
    ("dmma_small", _FEM6, dict(tc_slices=-1), _fp64, lambda p: _widest(p) <= 200),
    ("schur_h_wide", _W256, dict(tc_slices=-1), _fp64, lambda p: _widest(p) == 256 and _big_tiles(p) > 0),
    ("schur_h_wide", _W512, dict(tc_slices=-1), _fp64, lambda p: _widest(p) == 512 and _big_tiles(p) > 0),
    ("schur_h_wide_nolookahead", _W256, dict(tc_slices=-1, no_lookahead=1), _fp64, lambda p: _widest(p) == 256),
    ("schur_h_wide_nolookahead", _W512, dict(tc_slices=-1, no_lookahead=1), _fp64, lambda p: _widest(p) == 512),
    ("schur_h_narrow", _NARROW, dict(tc_slices=-1), _fp64, lambda p: _widest(p) <= 8 and _big_tiles(p) > 0),
    ("schur_h_many", _MANY, dict(tc_slices=-1), _fp64, lambda p: _big_tiles(p) > 0),
    ("strips512", _W2, dict(tc_slices=-1), _fp64, lambda p: _widest(p) == 512),   # _W512: 486 and 512 (above)
    ("default", _W256, dict(), _fp64, lambda p: _widest(p) == 256),
    ("default", _K2, dict(), _fp64, lambda p: _widest(p) == 256),
    ("pipeline", _W256, dict(pipeline=1), _fp64, lambda p: _widest(p) == 256),
]
CASES = [pytest.param(kw, opt, check, shape, E, id=f"{rid}-{_NAMES[id(kw)]}-E{E}")
         for rid, kw, opt, check, shape in ROUTES for E in (0, 10, 20)]
CASES += [pytest.param(kw, dict(tc_slices=s, tc_min_ns=64), _int8(s), lambda p: _widest(p) >= 128, 0,
                       id=f"int8_s{s}-{_NAMES[id(kw)]}-E0") for kw in (_K2, _K4) for s in (6, 7, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("kw,opt,check,shape,E", CASES)
def test_route_matches_oracle_entrywise(kw, opt, check, shape, E):
    info, st, prob, (lval, uval) = _factor_scaled(kw, E, **opt)
    assert shape(prob), "the problem does not have the shape this route needs"
    assert info == 0
    check(st)
    rl, ru = _reference(_NAMES[id(kw)], 0, False)
    el, eu = rel_err(lval, rl), rel_err(uval, ru)
    assert el < TOL and eu < TOL, (E, el, eu)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [_Z128, _Z200], ids=["z128", "z200"])
@pytest.mark.parametrize("E", [0, 10, 20])
def test_complex_matches_oracle_entrywise(kw, E):
    info, st, prob, (lval, uval) = _factor_scaled(kw, E, complex_=True)
    assert _widest(prob) >= 100
    assert info == 0
    _fp64(st)
    rl, ru = _reference(_NAMES[id(kw)], 0, True)
    el, eu = rel_err(lval, rl), rel_err(uval, ru)
    assert el < TOL and eu < TOL, (E, el, eu)


@pytest.mark.gpu
@pytest.mark.parametrize("E", [0, 10, 20])
def test_batched_members_match_oracle_entrywise(E):
    """Three members, each with its own values and its own row and column scales, on one batched handle (FP64)."""
    kw, B = _W256, 3
    rp, ci, v = pattern(kw)
    vals = [mixed_values(rp, ci, v, seed=20 + j) for j in range(B)]
    exps = [exponents(len(rp) - 1, E, seed=20 + j) for j in range(B)]
    prob, _ = poisson_problem(**kw)
    assert _widest(prob) == 256
    h = capi.BatchHandle(prob, B)
    h.fill_csr(rp, ci, np.stack([scaled(rp, ci, a, er, ec) for a, (er, ec) in zip(vals, exps)]), prob.perm)
    assert not h.factor().any()
    _fp64(h.stats())
    coords = panel_coords(prob, prob.layers[0])
    for j in range(B):
        h.download(j)
        er, ec = exps[j]
        lval, uval = unscale(prob, prob.layers[0], permuted(prob, er), permuted(prob, ec), coords)
        ref = make_problem(kw, vals[j])
        assert oracle.factor(ref)[0] == 0
        el, eu = rel_err(lval, ref.layers[0].lval), rel_err(uval, ref.layers[0].uval)
        assert el < TOL and eu < TOL, (j, E, el, eu)
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
@pytest.mark.parametrize("trans", ["N", "T"])
@pytest.mark.parametrize("E", [10, 20])
def test_solve_on_scaled_factors(complex_, trans, E):
    """A' x' = b' with b' = 2^er b gives x = 2^ec x'; A'^T x' = b' with b' = 2^ec b gives x = 2^er x': entry by entry
    against the solve on the unscaled matrix (the factored ordering throughout)."""
    kw = _Z128
    rp, ci, v = pattern(kw)
    vals = mixed_values(rp, ci, v, seed=7, complex_=complex_)
    er, ec = exponents(len(rp) - 1, E, seed=7)
    p0, p1 = make_problem(kw, vals), make_problem(kw, vals)
    h, hs = capi.Handle(p0, 0), capi.Handle(p1, 0)
    h.fill_csr(rp, ci, vals, p0.perm)
    hs.fill_csr(rp, ci, scaled(rp, ci, vals, er, ec), p1.perm)
    assert h.factor() == 0 and hs.factor() == 0
    er_p, ec_p = permuted(p0, er), permuted(p0, ec)
    bin_, bout = (er_p, ec_p) if trans == "N" else (ec_p, er_p)
    rng = np.random.default_rng(8)
    b = rng.standard_normal((2, p0.n))
    if complex_:
        b = b + 1j * rng.standard_normal((2, p0.n))
    x = h.solve(b, trans=trans)
    xs = ldexp(hs.solve(ldexp(b, bin_[None, :]), trans=trans), bout[None, :])
    assert np.abs(xs - x).max() <= 1e-12 * np.abs(x).max(), np.abs(xs - x).max() / np.abs(x).max()
    h.close()
    hs.close()
