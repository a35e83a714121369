"""slu_b200_inertia, _batch_inertia and _batch_fill_affine (and their slu_b200_z_ twins): eigenvalue counts of shifted
Laplacians, pencils and Hermitian matrices against the analytic spectrum, dense eigensolvers and oracle/inertia.py on the
downloaded factors; the tiny-pivot count against the factorization's own; Poisson 32^3 with wide supernodes; batched
against unbatched handles; affine fills bit for bit against host-built fills, also on batched Schur handles; and every
refusal.  The shifts are those test_inertia_cpu.py checks against the oracle."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sla

from oracle import inertia
from superlu_dist_b200 import capi
from test_gpu_schur import make as schur_make
from test_inertia_cpu import (BIG, BIG_WIDE, DEFECT_TOL, SHIFTS32, SMALL, TINY_SHIFTS, dense, diag_positions, flux_values,
                              gap_shifts, mass_values, rows_of, shifted, spectrum)
from test_scaled_parity import make_problem, panel_coords
from util import load_fixture, poisson_problem

pytestmark = pytest.mark.gpu
DTYPES = pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])


def pattern(kw):
    _, (rp, ci, v) = poisson_problem(**kw)
    return rp, ci, v


def gauge_values(rp, ci, v, seed=0):
    """D L D^H with D = diag(e^{i phi}): Hermitian, complex entries, the spectrum of the real L"""
    phi = np.random.default_rng(seed).uniform(-np.pi, np.pi, len(rp) - 1)
    return v * np.exp(1j * (phi[rows_of(rp)] - phi[np.asarray(ci)]))


def family(kw, complex_):
    """(rp, ci, base values, spectrum, shifts): the Laplacian in double, the random-flux Hermitian matrix in complex, with
    the shifts test_inertia_cpu.py checks on them"""
    rp, ci, v = pattern(kw)
    if not complex_:
        ev = spectrum(kw["N"])
        return rp, ci, v, ev, gap_shifts(ev, 7)
    a = flux_values(rp, ci, v, seed=kw["N"])
    ev = np.linalg.eigvalsh(dense(rp, ci, a))
    return rp, ci, a, ev, gap_shifts(ev, 5)


def unbatched_counts(kw, vals, perm=None):
    """inertia of one unbatched handle holding vals, and the restatement on its downloaded factors"""
    prob = make_problem(kw, vals)
    h = capi.Handle(prob, 0)
    h.fill_csr(*pattern(kw)[:2], vals, prob.perm if perm is None else perm)
    assert h.factor() == 0
    got = h.inertia()
    h.download()
    ref = inertia.inertia(prob, prob.layers[0])
    h.close()
    return got, ref


@pytest.mark.parametrize("kw", SMALL, ids=["poisson8", "poisson10"])
@DTYPES
def test_unbatched_counts(kw, complex_):
    rp, ci, a, ev, shifts = family(kw, complex_)
    n = len(rp) - 1
    for s in shifts:
        (neg, pos, tiny, defect), ref = unbatched_counts(kw, shifted(rp, ci, a, s))
        assert (neg, pos, tiny) == (int(np.sum(ev < s)), n - int(np.sum(ev < s)), 0), s
        assert (neg, pos, tiny) == ref[:3] and abs(defect - ref[3]) <= 1e-15
        assert defect <= DEFECT_TOL if complex_ else defect == 0.0


def test_non_hermitian_complex_defect():
    kw = SMALL[0]
    rp, ci, v = pattern(kw)
    a = shifted(rp, ci, v, 0.5) + 0j
    a[rows_of(rp) == np.asarray(ci)] += 0.25j
    (neg, pos, _, defect), ref = unbatched_counts(kw, a)
    assert defect > 1e-3 and abs(defect - ref[3]) <= 1e-12 and (neg, pos) == ref[:2]


@pytest.mark.parametrize("sigma", TINY_SHIFTS)
def test_tiny_equals_factorization_count(sigma):
    prob, _, _ = load_fixture("poisson12_nd_tiny")
    lay = prob.layers[0]
    lay.lval[diag_positions(prob, lay)] -= sigma
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    neg, pos, tiny, _ = h.inertia()
    assert tiny == h.stats().tiny_pivots and neg + pos == prob.n
    h.download()
    assert (neg, pos, tiny) == inertia.inertia(prob, lay)[:3]
    if sigma:
        assert tiny > 0
    h.close()


def test_batched_tiny_sums_to_stats():
    """Members of the tiny-pivot fixture's pattern with replacement on: the per-member counts sum to stats.tiny_pivots"""
    kw = dict(N=12, leaf=16, relax=6, maxsup=24)
    rp, ci, v = pattern(kw)
    vals = np.stack([shifted(rp, ci, v, s) for s in (4.0, 0.5, 5.0)])
    prob = make_problem(kw, vals[0])
    prob.replace_tiny_pivot, prob.thresh = 1, 7.152557373046875e-07
    bh = capi.BatchHandle(prob, 3)
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    neg, pos, tiny, _ = bh.inertia()
    assert int(tiny.sum()) == bh.stats().tiny_pivots and np.all(neg + pos == prob.n)
    bh.close()


@pytest.mark.parametrize("complex_", [False, True], ids=["double_w512", "complex_w256"])
def test_poisson32_at_scale(complex_):
    """Shifts among the lowest 400 eigenvalues of Poisson 32^3; in complex the gauge-transformed Laplacian D L D^H"""
    kw = BIG if complex_ else BIG_WIDE
    rp, ci, v = pattern(kw)
    a = gauge_values(rp, ci, v) if complex_ else v
    ev = spectrum(32)
    vals = np.stack([shifted(rp, ci, a, s) for s in SHIFTS32])
    prob = make_problem(kw, vals[0])
    assert np.diff(np.asarray(prob.xsup)).max() == kw["maxsup"]
    want = np.array([int(np.sum(ev < s)) for s in SHIFTS32])
    bh = capi.BatchHandle(prob, len(SHIFTS32))
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    neg, pos, tiny, defect = bh.inertia()
    assert np.array_equal(neg, want) and np.all(pos == prob.n - want) and not tiny.any()
    assert np.all(defect <= DEFECT_TOL) if complex_ else not defect.any()
    h = capi.Handle(prob, 0)
    for j in (0, len(SHIFTS32) - 1):
        h.fill_csr(rp, ci, vals[j], prob.perm)
        assert h.factor() == 0
        assert h.inertia()[:3] == (want[j], prob.n - want[j], 0)
    h.close()
    bh.close()


@pytest.mark.parametrize("B", [1, 7, 64])
@DTYPES
def test_batched_against_unbatched(B, complex_):
    kw = SMALL[0]
    rp, ci, a, ev, shifts = family(kw, complex_)
    sig = [shifts[j % len(shifts)] for j in range(B)]
    vals = np.stack([shifted(rp, ci, a, s) for s in sig])
    prob = make_problem(kw, vals[0])
    bh = capi.BatchHandle(prob, B)
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    neg, pos, tiny, defect = bh.inertia()
    assert neg.shape == pos.shape == tiny.shape == defect.shape == (B,)
    one = {}
    for j, s in enumerate(sig):
        if s not in one:
            one[s] = unbatched_counts(kw, vals[j], prob.perm)[0]
        got = one[s]
        assert (neg[j], pos[j], tiny[j]) == got[:3] and neg[j] == int(np.sum(ev < s))
        assert defect[j] <= DEFECT_TOL and got[3] <= DEFECT_TOL
    bh.close()


def arena(bh, j):
    bh.download(j)
    lay = bh.prob.layers[0]
    return lay.lval.copy(), lay.uval.copy()


def same_arenas(b1, b2, members):
    for j in members:
        (l1, u1), (l2, u2) = arena(b1, j), arena(b2, j)
        assert np.array_equal(l1, l2) and np.array_equal(u1, u2), j


def test_pencil_fill_affine():
    """fill_affine(K, M; 1, -sigma_j) + batch_factor + batch_inertia against eigh(K, M); the fill bit for bit against the
    host-built K - sigma_j M through batch_fill_csr, before factoring"""
    kw = SMALL[1]
    rp, ci, v = pattern(kw)
    m = mass_values(rp, ci)
    ev = sla.eigh(dense(rp, ci, v), dense(rp, ci, m), eigvals_only=True)
    shifts = gap_shifts(ev, 5)
    coef = np.array([[1.0, -s] for s in shifts])
    prob = make_problem(kw, v)
    ba, bc = capi.BatchHandle(prob, len(shifts)), capi.BatchHandle(prob, len(shifts))
    ba.fill_affine(rp, ci, np.stack([v, m]), coef, prob.perm)
    bc.fill_csr(rp, ci, np.stack([shifted(rp, ci, v, s, m) for s in shifts]), prob.perm)
    same_arenas(ba, bc, (0, len(shifts) - 1))
    assert not ba.factor().any()
    neg, pos, tiny, _ = ba.inertia()
    assert np.array_equal(neg, [int(np.sum(ev < s)) for s in shifts]) and not tiny.any()
    ba.close()
    bc.close()


@DTYPES
def test_fill_affine_bit_exact_and_general(complex_):
    kw = SMALL[0]
    rp, ci, v = pattern(kw)
    m, c = mass_values(rp, ci), 0.5 * mass_values(rp, ci)
    B = 6
    dt = np.complex128 if complex_ else np.float64
    prob = make_problem(kw, v.astype(dt))
    ba, bc = capi.BatchHandle(prob, B), capi.BatchHandle(prob, B)
    # T = 1, coef 1: the batch_fill_csr route
    ba.fill_affine(rp, ci, v[None, :], np.ones((B, 1)), prob.perm)
    bc.fill_csr(rp, ci, np.stack([v] * B), prob.perm)
    same_arenas(ba, bc, (0, B - 1))
    # dyadic coefficients: T = 2 (K - sigma M), and in complex T = 3 (K - w^2 M + i w C)
    w = np.arange(1, B + 1) / 8.0
    if complex_:
        terms, coef = np.stack([v, m, c]), np.stack([np.ones(B), -w * w, 1j * w], axis=1)
        host = np.stack([v - wj * wj * m + 1j * wj * c for wj in w])
    else:
        terms, coef = np.stack([v, m]), np.stack([np.ones(B), -w], axis=1)
        host = np.stack([v - wj * m for wj in w])
    ba.fill_affine(rp, ci, terms, coef, prob.perm)
    bc.fill_csr(rp, ci, host, prob.perm)
    same_arenas(ba, bc, range(B))
    # general coefficients: within one rounding per term, then equal counts and factors within 1e-12
    rng = np.random.default_rng(3)
    coef = np.stack([np.ones(B), -rng.uniform(0.1, 3.0, B), 0.5 * rng.uniform(-1, 1, B)], axis=1).astype(dt)
    if complex_:
        coef[:, 2] *= 1j
    terms = np.stack([v, m, c]).astype(dt)
    host = coef @ terms
    ba.fill_affine(rp, ci, terms, coef, prob.perm)
    bc.fill_csr(rp, ci, host, prob.perm)
    bound = 8 * np.finfo(np.float64).eps * (np.abs(coef) @ np.abs(terms)).max()
    for j in (0, B - 1):
        (l1, u1), (l2, u2) = arena(ba, j), arena(bc, j)
        assert np.abs(l1 - l2).max() <= bound and np.abs(u1 - u2).max(initial=0) <= bound
    assert not ba.factor().any() and not bc.factor().any()
    ia, ic = ba.inertia(), bc.inertia()
    for q in range(3):
        assert np.array_equal(ia[q], ic[q])
    for j in (0, B - 1):
        (l1, u1), (l2, u2) = arena(ba, j), arena(bc, j)
        assert np.abs(l1 - l2).max() <= 1e-12 * np.abs(l2).max() and np.abs(u1 - u2).max(initial=0) <= 1e-12 * np.abs(u2).max()
    ba.close()
    bc.close()


@DTYPES
def test_fill_affine_on_batched_schur_handle(complex_):
    prob, (rp, ci, vals), s, _ = schur_make("p8_top", np.complex128 if complex_ else np.float64, dense=False)
    m = mass_values(rp, ci)
    sig = [-0.5, -0.25, -0.125]
    ba, bc = capi.BatchSchurHandle(prob, 3, s), capi.BatchSchurHandle(prob, 3, s)
    ba.fill_affine(rp, ci, np.stack([vals, m]), np.array([[1.0, -x] for x in sig]), prob.perm)
    bc.fill_csr(rp, ci, np.stack([vals - x * m for x in sig]), prob.perm)
    same_arenas(ba, bc, range(3))
    assert not ba.factor().any() and not bc.factor().any()
    Sa, Sc = ba.schur(), bc.schur()
    assert np.abs(Sa - Sc).max() <= 1e-12 * np.abs(Sc).max()
    with pytest.raises(RuntimeError, match="batch_inertia on a Schur handle"):
        ba.inertia()
    ba.close()
    bc.close()


@DTYPES
def test_refusals(complex_):
    L = capi.lib()
    z = "z_" if complex_ else ""
    fn = lambda name: getattr(L, f"slu_b200_{z}{name}")  # noqa: E731
    err = lambda: L.slu_b200_last_error()  # noqa: E731
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    rp, ci, v = pattern(kw)
    dt = np.complex128 if complex_ else np.float64
    vals = np.stack([shifted(rp, ci, v, 0.25 * j) for j in range(3)]).astype(dt)
    prob = make_problem(kw, vals[0])
    n, perm = prob.n, np.asarray(prob.perm, np.int32)
    cnt, dfc = (C.c_int64 * 9)(), (C.c_double * 3)()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    terms, coef = vals[:1].copy(), np.ones((3, 1), dt)
    # unbatched handle: inertia before factor, then fill_affine / batch_inertia refused
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="inertia needs a successful"):
        h.inertia()
    h.fill_csr(rp, ci, vals[0], perm)
    assert h.factor() == 0
    assert fn("batch_inertia")(h.h, cnt, dfc) < 0 and b"unbatched handle" in err()
    assert fn("batch_fill_affine")(h.h, n, vp(rp), vp(ci), 1, vp(terms), vp(coef), vp(perm)) < 0 and b"unbatched handle" in err()
    assert h.inertia()[:2] == (0, n)                       # still usable
    h.close()
    # unbatched Schur handle
    sp_, (srp, sci, svals), s, _ = schur_make("p8_top", dt, dense=False)
    sh = capi.SchurHandle(sp_, s)
    sh.fill_csr(srp, sci, svals, sp_.perm)
    assert sh.factor() == 0
    with pytest.raises(RuntimeError, match="inertia on a Schur handle"):
        sh.inertia()
    sh.close()
    # batched handle
    bh = capi.BatchHandle(prob, 3)
    with pytest.raises(RuntimeError, match="batch_inertia needs a .*batch_factor"):
        bh.inertia()
    assert fn("inertia")(bh.h, cnt, dfc) < 0 and b"batched handle" in err()
    args = lambda **k: dict(dict(n=n, rp=rp, ci=ci, T=1, terms=terms, coef=coef, perm=perm), **k)  # noqa: E731

    def call(a):
        return fn("batch_fill_affine")(bh.h, a["n"], vp(a["rp"]) if a["rp"] is not None else None, vp(a["ci"]), a["T"],
                                       vp(a["terms"]), vp(a["coef"]), vp(a["perm"]))
    assert call(args(T=0)) < 0 and b"nterms = 0" in err()
    assert call(args(n=n - 1)) < 0 and b"does not match" in err()
    assert call(args(rp=None)) < 0 and b"null argument" in err()
    bad = rp.copy()
    bad[3] = bad[4] + 1
    assert call(args(rp=bad)) < 0 and b"bad rowptr" in err()
    bad = ci.copy()
    bad[5] = n
    assert call(args(ci=bad)) < 0 and b"outside" in err()
    # an entry with no slot: one entry (0, c0) of A whose (perm[0], perm[c0]) is not stored in L + U
    lrow, lcol, urow, ucol = panel_coords(prob, prob.layers[0])
    slots = set(zip(lrow.tolist(), lcol.tolist())) | set(zip(urow[urow >= 0].tolist(), ucol[urow >= 0].tolist()))
    c0 = next(c for c in range(n) if (perm[0], perm[c]) not in slots)
    rp1 = np.array([0] + [1] * n, np.int32)
    ci1 = np.array([c0], np.int32)
    t1 = np.ones((1, 1), dt)
    assert call(args(rp=rp1, ci=ci1, terms=t1)) < 0 and b"1 entries of the pattern have no slot" in err()
    # a good fill, then batch_solve fails until batch_factor
    bh.fill_affine(rp, ci, terms, coef, perm)
    with pytest.raises(RuntimeError, match="batch_factor"):
        bh.solve(np.ones((3, n), dt))
    assert not bh.factor().any()
    assert bh.inertia()[0].shape == (3,)
    bh.solve(np.ones((3, n), dt))
    # member 1 with an exact zero pivot
    vz = vals.copy()
    vz[1, perm[ci] == 0] = 0.0
    bh.fill_csr(rp, ci, vz, perm)
    info = bh.factor()
    assert info[1] == 1
    with pytest.raises(RuntimeError, match="batch_inertia: member 1 has an exact zero pivot"):
        bh.inertia()
    bh.close()
