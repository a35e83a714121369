"""slu_b200_z_selinv, slu_b200_z_selinv_get and slu_b200_z_logdet on the resident doublecomplex factors: H = F^-T (a
plain transpose) on the stored pattern of L + U against a dense inverse and against oracle/selinv.py run on the GPU's own
downloaded factors, a complex-symmetric shifted matrix, an exact phase rotation, exact power-of-two scaling, unit-vector
solves, determinism, untouched factors, the launch count and every refusal."""
import ctypes as C

import numpy as np
import pytest

from oracle import selinv
from superlu_dist_b200 import capi
from test_gpu_selinv import csr_of, factored_handle, stored_positions
from test_gpu_solve_complex import complex_csr
from test_scaled_parity import exponents, ldexp, make_problem, mixed_values, scaled
from test_selinv_complex_cpu import complex_logdet, shifted_problem
from util import complex_problem, load_fixture, poisson_problem

pytestmark = pytest.mark.gpu
TOL = 1e-10
GENERATED = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=5, leaf=4, relax=8, maxsup=200, fem=3),
             dict(N=10, leaf=8, relax=16, maxsup=128)]


def gpu_h(h, prob, rows, cols):
    """H(rows, cols) read back through inv_entries with the identity permutation: A^-1(i, j) = H(j, i)"""
    rp, ci, order = csr_of(cols, rows, prob.n)
    vals = h.inv_entries(rp, ci, np.arange(prob.n, dtype=np.int32))
    assert vals.dtype == np.complex128
    out = np.empty(len(rows), np.complex128)
    out[order] = vals
    return out


def check_h(got, ref, rows, cols):
    scale = np.abs(ref).max()
    assert np.abs(got - ref).max() <= TOL * scale, np.abs(got - ref).max() / scale
    dg = rows == cols
    assert np.all(np.abs(got[dg] - ref[dg]) <= TOL * np.abs(ref[dg]))


def check_dense(prob, h):
    """H from the GPU against inv(L U)^T of the downloaded factors; the log-determinant against numpy.linalg.slogdet"""
    lay = prob.layers[0]
    out = h.selinv()
    assert out[0] > 0 and out[1] > 0 and out[3] >= 16 * (len(lay.lval) - 1)
    L, U = prob.dense(lay, True)
    G = np.linalg.inv(L @ U)
    rows, cols, _ = stored_positions(prob, lay)
    check_h(gpu_h(h, prob, rows, cols), G.T[rows, cols], rows, cols)
    sign, logabs = h.logdet()
    s2, l2 = np.linalg.slogdet(L @ U)
    assert isinstance(sign, complex) and abs(abs(sign) - 1.0) <= 1e-14
    assert abs(sign - s2) <= 1e-12 and abs(logabs - l2) <= 1e-12 * max(1.0, abs(l2))
    return G


SMALL = [pytest.param(lambda: load_fixture("cg20_pzdrive3d")[0], id="cg20_pzdrive3d")] + \
        [pytest.param(lambda kw=kw: complex_problem(**kw), id=f"gen{i}") for i, kw in enumerate(GENERATED)]


@pytest.mark.parametrize("make", SMALL)
def test_z_selinv_against_dense_inverse(make):
    prob = make()
    h = factored_handle(prob)
    check_dense(prob, h)
    h.close()


@pytest.mark.parametrize("kw", [GENERATED[0], GENERATED[2]], ids=["poisson8", "poisson10"])
def test_z_selinv_complex_symmetric_shift(kw):
    """A = K - (E + i eta) I, eta = 0.5: A^-1 is complex symmetric and not Hermitian.  inv_entries on the pattern of A
    (with A's own permutation) is symmetric to TOL and differs from its conjugate transpose."""
    prob, rp, ci, vals = shifted_problem(kw)
    h = factored_handle(prob)
    check_dense(prob, h)
    n = prob.n
    rows = np.repeat(np.arange(n), np.diff(rp))
    g = h.inv_entries(rp, ci, prob.perm)              # A^-1(rows, ci), CSR order
    gt = np.empty_like(g)
    pos = {(int(r), int(c)): p for p, (r, c) in enumerate(zip(rows, ci))}
    for p, (r, c) in enumerate(zip(rows, ci)):
        gt[p] = g[pos[(int(c), int(r))]]              # A^-1(ci, rows)
    scale = np.abs(g).max()
    assert np.abs(g - gt).max() <= TOL * scale
    assert np.abs(g - gt.conj()).max() > 1e-3 * scale
    h.close()


BIG = [dict(N=16, leaf=16, relax=32, maxsup=256), dict(N=32, leaf=16, relax=32, maxsup=256),
       dict(N=16, leaf=16, relax=32, maxsup=256, fem=3)]


@pytest.mark.parametrize("kw", BIG, ids=["p16_w256", "p32", "fem16"])
def test_z_selinv_against_oracle_on_gpu_factors(kw):
    prob = complex_problem(**kw)
    if kw["N"] == 16 and not kw.get("fem"):
        assert np.diff(np.asarray(prob.xsup)).max() == 256      # the z supernode cap is reached
    h = factored_handle(prob)
    lay = prob.layers[0]
    h.selinv()
    hl, hu = selinv.selinv(prob, lay)
    rows, cols, u = stored_positions(prob, lay)
    check_h(gpu_h(h, prob, rows, cols), np.concatenate([hl, hu[u]]), rows, cols)
    sign, logabs = h.logdet()
    s2, l2 = complex_logdet(prob, lay)
    assert abs(sign - s2) <= 1e-12 and abs(logabs - l2) <= 1e-12 * abs(l2)
    st = h.stats()
    assert h.selinv()[2] == 7 * st.nlevels - 1      # one tree: every level but the root's has a Schur update to map
    h.close()


def _rotated_fixture(name, phi):
    """The fixture's matrix times exp(i phi), as a complex layer (complex_problem's construction from a real one)"""
    prob = load_fixture(name)[0]
    prob.dtype = np.dtype(np.complex128)
    for lay in prob.layers.values():
        lay.lval = lay.lval.astype(np.complex128) * np.exp(1j * phi)
        lay.uval = lay.uval.astype(np.complex128) * np.exp(1j * phi)
    return prob


def test_z_selinv_phase_rotation():
    """F' = exp(i phi) F on unsym360_mmd (unsymmetric pattern, zero-padded U columns): H' = exp(-i phi) H, log |det|
    unchanged and sign' = exp(i n phi) sign."""
    phi = 0.3
    p0, p1 = _rotated_fixture("unsym360_mmd", 0.0), _rotated_fixture("unsym360_mmd", phi)
    h0, h1 = factored_handle(p0), factored_handle(p1)
    h0.selinv()
    h1.selinv()
    rows, cols, _ = stored_positions(p0, p0.layers[0])
    a0, a1 = gpu_h(h0, p0, rows, cols), gpu_h(h1, p1, rows, cols)
    check_h(a1, np.exp(-1j * phi) * a0, rows, cols)
    s0, l0 = h0.logdet()
    s1, l1 = h1.logdet()
    assert abs(l1 - l0) <= 1e-12 * abs(l0)
    assert abs(s1 - np.exp(1j * p0.n * phi) * s0) <= TOL
    h0.close()
    h1.close()


@pytest.mark.parametrize("E", [0, 10, 20])
def test_z_scaled_inverse_and_logdet(E):
    """A' = 2^er A 2^ec: A'^-1 = 2^-ec A^-1 2^-er entry by entry, log |det A'| = log |det A| + (sum er + sum ec) ln 2."""
    kw = dict(N=10, leaf=8, relax=16, maxsup=128)
    _, (rp, ci, v) = poisson_problem(**kw)
    vals = mixed_values(rp, ci, v, seed=9, complex_=True)
    n = len(rp) - 1
    er, ec = exponents(n, E, seed=9)
    prob0, prob1 = make_problem(kw, vals), make_problem(kw, vals)
    h0, h1 = capi.Handle(prob0, 0), capi.Handle(prob1, 0)
    h0.fill_csr(rp, ci, vals, prob0.perm)
    h1.fill_csr(rp, ci, scaled(rp, ci, vals, er, ec), prob1.perm)
    assert h0.factor() == 0 and h1.factor() == 0
    h0.selinv()
    h1.selinv()
    rows, cols, _ = stored_positions(prob0, prob0.layers[0])
    iperm = np.argsort(prob0.perm)
    ai, aj = iperm[cols], iperm[rows]
    prp, pci, order = csr_of(ai, aj, n)
    g0 = h0.inv_entries(prp, pci, prob0.perm)
    g1 = ldexp(h1.inv_entries(prp, pci, prob1.perm), ec[ai[order]] + er[aj[order]])
    assert np.abs(g1 - g0).max() <= TOL * np.abs(g0).max()
    dg = ai[order] == aj[order]
    assert np.all(np.abs(g1[dg] - g0[dg]) <= TOL * np.abs(g0[dg]))
    s0, l0 = h0.logdet()
    s1, l1 = h1.logdet()
    A = np.zeros((n, n), np.complex128)
    A[np.repeat(np.arange(n), np.diff(rp)), ci] = vals
    sd, ld = np.linalg.slogdet(A)
    assert abs(s0 - sd) <= 1e-12 and abs(s1 - s0) <= 1e-14 and abs(l0 - ld) <= 1e-12 * abs(ld)
    shift = (er.sum() + ec.sum()) * np.log(2.0)
    assert abs(l1 - (l0 + shift)) <= 1e-12 * abs(l0 + shift)
    h0.close()
    h1.close()


def test_z_poisson32_columns_by_solves():
    """16 columns of F^-1 (A = F: identity permutation) from unit-vector z_solve calls against inv_entries."""
    prob = complex_problem(N=32, leaf=16, relax=32, maxsup=256)
    n = prob.n
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    h.selinv()
    rows, cols, _ = stored_positions(prob, prob.layers[0])
    for j in np.random.default_rng(5).choice(n, 16, replace=False):
        e = np.zeros(n, np.complex128)
        e[j] = 1.0
        x = h.solve(e)                               # column j of F^-1
        i = cols[rows == j]                          # H(j, i) = F^-1(i, j) is stored
        rp, ci, order = csr_of(i, np.full(len(i), j), n)
        got = np.empty(len(i), np.complex128)
        got[order] = h.inv_entries(rp, ci, np.arange(n, dtype=np.int32))
        assert np.abs(got - x[i]).max() <= TOL * np.abs(x).max()
    h.close()


def test_z_deterministic_and_factors_untouched():
    prob = complex_problem(N=16, leaf=16, relax=32, maxsup=256)
    h = factored_handle(prob)
    lay = prob.layers[0]
    l0, u0 = lay.lval.copy(), lay.uval.copy()
    rng = np.random.default_rng(6)
    b = rng.standard_normal(prob.n) + 1j * rng.standard_normal(prob.n)
    x0 = h.solve(b)
    h.selinv()
    rows, cols, _ = stored_positions(prob, lay)
    a = gpu_h(h, prob, rows, cols)
    h.selinv()
    assert np.array_equal(a, gpu_h(h, prob, rows, cols))
    d1 = h.inv_diag()
    assert np.array_equal(d1, a[rows == cols][np.argsort(rows[rows == cols])])
    h.download()
    assert np.array_equal(lay.lval, l0) and np.array_equal(lay.uval, u0)
    x1 = h.solve(b)
    # the solve accumulates with atomics, whose order is not fixed: equal up to the last bits
    assert np.abs(x1 - x0).max() <= 1e-14 * np.abs(x0).max()
    h.close()


def test_z_refusals():
    L = capi.lib()
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    prob = complex_problem(**kw)
    rp, ci, v = complex_csr(**kw)
    n = prob.n
    out = (C.c_double * 4)()
    ident = np.arange(n, dtype=np.int32)
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="slu_b200_z_selinv needs a successful"):
        h.selinv()                                    # before factor
    with pytest.raises(RuntimeError, match="needs a successful"):
        h.logdet()
    h.upload()
    assert h.factor() == 0
    with pytest.raises(RuntimeError, match="selinv on the current factors"):
        h.inv_diag()                                  # _get before selinv
    h.selinv()
    assert np.isfinite(h.inv_diag()).all()
    # wrong n
    rp1 = np.arange(n, dtype=np.int32)
    assert L.slu_b200_z_selinv_get(h.h, n - 1, rp1.ctypes.data_as(C.c_void_p), rp1.ctypes.data_as(C.c_void_p),
                                   ident.ctypes.data_as(C.c_void_p), (C.c_double * (2 * n))()) < 0
    assert b"does not match" in L.slu_b200_last_error()
    # an entry with no slot in L + U
    rows, cols, _ = stored_positions(prob, prob.layers[0])
    have = set(zip(rows.tolist(), cols.tolist()))
    r, c = next((r, c) for r in range(n) for c in range(n) if (r, c) not in have)
    with pytest.raises(RuntimeError, match="1 entries have no slot"):
        h.inv_entries(np.array([0] * (c + 1) + [1] * (n - c), np.int32), np.array([r], np.int32), ident)
    # a refactor invalidates the inverse
    h.upload()
    assert h.factor() == 0
    with pytest.raises(RuntimeError, match="selinv on the current factors"):
        h.inv_diag()
    h.close()
    # info > 0: column 0 of F = P A P^T is zero
    vz = np.array(v, np.complex128)
    vz[np.asarray(prob.perm)[ci] == 0] = 0.0
    hz = capi.Handle(prob, 0)
    hz.fill_csr(rp, ci, vz, prob.perm)
    assert hz.factor() == 1
    with pytest.raises(RuntimeError, match="needs a successful"):
        hz.selinv()
    hz.close()
    # batched doublecomplex handle
    bh = capi.BatchHandle(prob, 2)
    bh.fill_csr(rp, ci, np.stack([v, v]), prob.perm)
    assert not bh.factor().any()
    assert L.slu_b200_z_selinv(bh.h, out) < 0 and b"batched handle" in L.slu_b200_last_error()
    la, sg = C.c_double(), (C.c_double * 2)()
    assert L.slu_b200_z_logdet(bh.h, C.byref(la), sg) < 0 and b"batched handle" in L.slu_b200_last_error()
    bh.close()
