"""slu_b200_selinv, slu_b200_selinv_get and slu_b200_logdet on the resident factors: H = F^-T on the stored pattern of
L + U against a dense inverse and against oracle/selinv.py run on the GPU's own downloaded factors, unit-vector solves,
determinism, untouched factors, exact power-of-two scaling, and every refusal."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle, selinv
from superlu_dist_b200 import capi
from test_gpu_solve_trans import CASES, real_case, unsym_values
from test_scaled_parity import exponents, ldexp, mixed_values, panel_coords, scaled
from util import load_fixture, poisson_problem

pytestmark = pytest.mark.gpu
TOL = 1e-10
FIXTURES = ["g4_pddrive3d", "g20_pddrive3d", "poisson8_nd", "poisson12_nd_tiny", "fem5_mmd", "unsym360_mmd"]
GENERATED = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=5, leaf=4, relax=8, maxsup=200, fem=3),
             dict(N=10, leaf=8, relax=16, maxsup=128)]


def stored_positions(prob, lay):
    """(rows, cols) in the factored ordering of every stored value of L and U, in the order of layer.lval then layer.uval"""
    lrow, lcol, urow, ucol = panel_coords(prob, lay)
    u = urow >= 0
    return np.concatenate([lrow, urow[u]]), np.concatenate([lcol, ucol[u]]), u


def csr_of(i, j, n):
    """CSR pattern of the pairs (i, j) -> (rowptr, colind, order) with colind = j[order]"""
    order = np.lexsort((j, i))
    rp = np.concatenate([[0], np.cumsum(np.bincount(i, minlength=n))]).astype(np.int32)
    return rp, j[order].astype(np.int32), order


def gpu_h(h, prob, rows, cols):
    """H(rows, cols) read back through inv_entries with the identity permutation: A^-1(i, j) = H(j, i)"""
    rp, ci, order = csr_of(cols, rows, prob.n)
    vals = h.inv_entries(rp, ci, np.arange(prob.n, dtype=np.int32))
    out = np.empty(len(rows))
    out[order] = vals
    return out


def factored_handle(prob):
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    h.download()                     # the factors the GPU made, into prob.layers[0]
    return h


def check_h(got, ref, rows, cols):
    scale = np.abs(ref).max()
    assert np.abs(got - ref).max() <= TOL * scale, np.abs(got - ref).max() / scale
    dg = rows == cols
    assert np.all(np.abs(got[dg] - ref[dg]) <= TOL * np.abs(ref[dg]))


def _fixture(name):
    return load_fixture(name)[0]


def _generated(kw, values):
    prob, (rp, ci, v) = poisson_problem(**kw)
    prob.fill_layer(0, rp, ci, unsym_values(rp, ci, v) if values == "unsym" else mixed_values(rp, ci, v, seed=3))
    return prob


SMALL = [pytest.param(lambda n=n: _fixture(n), id=n) for n in FIXTURES] + \
        [pytest.param(lambda kw=kw, v=v: _generated(kw, v), id=f"{i}-{v}") for i, kw in enumerate(GENERATED) for v in ("unsym", "mixed")]


@pytest.mark.parametrize("make", SMALL)
def test_selinv_against_dense_inverse(make):
    prob = make()
    h = factored_handle(prob)
    lay = prob.layers[0]
    out = h.selinv()
    assert out[0] > 0 and out[1] > 0 and out[3] >= 8 * (len(lay.lval) - 1)
    L, U = prob.dense(lay, True)
    G = np.linalg.inv(L @ U)
    rows, cols, _ = stored_positions(prob, lay)
    check_h(gpu_h(h, prob, rows, cols), G.T[rows, cols], rows, cols)
    sign, logabs = h.logdet()
    s2, l2 = np.linalg.slogdet(L @ U)
    assert sign == s2 and abs(logabs - l2) <= 1e-12 * max(1.0, abs(l2))
    h.close()


BIG = CASES + [dict(N=32, leaf=16, relax=32, maxsup=256), dict(N=16, leaf=16, relax=32, maxsup=256, fem=3)]


@pytest.mark.parametrize("kw", BIG, ids=["p8", "p12", "fem5", "p16_w256", "fem18_w512", "p32", "fem16"])
def test_selinv_against_oracle_on_gpu_factors(kw):
    prob = real_case(kw)[0]
    if kw["maxsup"] >= 256:
        assert np.diff(np.asarray(prob.xsup)).max() == kw["maxsup"]
    h = factored_handle(prob)
    lay = prob.layers[0]
    h.selinv()
    hl, hu = selinv.selinv(prob, lay)
    rows, cols, u = stored_positions(prob, lay)
    check_h(gpu_h(h, prob, rows, cols), np.concatenate([hl, hu[u]]), rows, cols)
    sign, logabs = h.logdet()
    s2, l2 = selinv.logdet(prob, lay)
    assert sign == s2 and abs(logabs - l2) <= 1e-12 * abs(l2)
    st = h.stats()
    assert h.selinv()[2] == 7 * st.nlevels - 1      # one tree: every level but the root's has a Schur update to map
    h.close()


def test_poisson48_columns_by_solves():
    """16 columns of A^-1 (A = F here: identity permutation) from unit-vector solves against inv_entries on the entries
    of H those columns meet."""
    prob = real_case(dict(N=48, leaf=16, relax=32, maxsup=256))[0]
    n = prob.n
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    h.selinv()
    rows, cols, _ = stored_positions(prob, prob.layers[0])
    for j in np.random.default_rng(5).choice(n, 16, replace=False):
        e = np.zeros(n)
        e[j] = 1.0
        x = h.solve(e)                               # column j of F^-1
        i = cols[rows == j]                          # H(j, i) = F^-1(i, j) is stored
        rp, ci, order = csr_of(i, np.full(len(i), j), n)
        got = np.empty(len(i))
        got[order] = h.inv_entries(rp, ci, np.arange(n, dtype=np.int32))
        assert np.abs(got - x[i]).max() <= TOL * np.abs(x).max()
    h.close()


def test_deterministic_and_factors_untouched():
    kw = CASES[3]
    prob = real_case(kw)[0]
    h = factored_handle(prob)
    lay = prob.layers[0]
    l0, u0 = lay.lval.copy(), lay.uval.copy()
    b = np.random.default_rng(6).standard_normal(prob.n)
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


@pytest.mark.parametrize("E", [0, 10, 20])
def test_scaled_inverse_and_logdet(E):
    """A' = 2^er A 2^ec: A'^-1 = 2^-ec A^-1 2^-er entry by entry, log |det A'| = log |det A| + (sum er + sum ec) ln 2."""
    kw = dict(N=10, leaf=8, relax=16, maxsup=128)
    prob0, (rp, ci, v) = poisson_problem(**kw)
    n = prob0.n
    vals = mixed_values(rp, ci, v, seed=9)
    er, ec = exponents(n, E, seed=9)
    prob1, _ = poisson_problem(**kw)
    h0, h1 = capi.Handle(prob0, 0), capi.Handle(prob1, 0)
    h0.fill_csr(rp, ci, vals, prob0.perm)
    h1.fill_csr(rp, ci, scaled(rp, ci, vals, er, ec), prob1.perm)
    assert h0.factor() == 0 and h1.factor() == 0
    h0.selinv()
    h1.selinv()
    # every stored position of H as an entry of A^-1: H(r, c) = A^-1(iperm[c], iperm[r])
    rows, cols, _ = stored_positions(prob0, prob0.layers[0])
    iperm = np.argsort(prob0.perm)
    ai, aj = iperm[cols], iperm[rows]
    prp, pci, order = csr_of(ai, aj, n)
    g0 = h0.inv_entries(prp, pci, prob0.perm)
    g1 = ldexp(h1.inv_entries(prp, pci, prob1.perm), ec[ai[order]] + er[aj[order]])
    assert np.abs(g1 - g0).max() <= TOL * np.abs(g0).max()
    s0, l0 = h0.logdet()
    s1, l1 = h1.logdet()
    A = np.zeros((n, n))
    A[np.repeat(np.arange(n), np.diff(rp)), ci] = vals
    sd, ld = np.linalg.slogdet(A)
    assert s0 == sd == s1 and abs(l0 - ld) <= 1e-12 * abs(ld)
    shift = (er.sum() + ec.sum()) * np.log(2.0)
    assert abs(l1 - (l0 + shift)) <= 1e-12 * abs(l0 + shift)
    h0.close()
    h1.close()


def test_refusals():
    L = capi.lib()
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    prob, (rp, ci, v) = poisson_problem(**kw)
    n = prob.n
    out = (C.c_double * 4)()
    ident = np.arange(n, dtype=np.int32)
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="needs a successful"):
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
    assert L.slu_b200_selinv_get(h.h, n - 1, rp1.ctypes.data_as(C.c_void_p), rp1.ctypes.data_as(C.c_void_p),
                                 ident.ctypes.data_as(C.c_void_p), (C.c_double * n)()) < 0
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
    vz = np.array(v, np.float64)
    vz[np.asarray(prob.perm)[ci] == 0] = 0.0
    hz = capi.Handle(prob, 0)
    hz.fill_csr(rp, ci, vz, prob.perm)
    assert hz.factor() == 1
    with pytest.raises(RuntimeError, match="needs a successful"):
        hz.selinv()
    hz.close()
    # batched handle
    bh = capi.BatchHandle(prob, 2)
    bh.fill_csr(rp, ci, np.stack([v, v]), prob.perm)
    assert not bh.factor().any()
    assert L.slu_b200_selinv(bh.h, out) < 0 and b"batched handle" in L.slu_b200_last_error()
    la, sg = C.c_double(), C.c_double()
    assert L.slu_b200_logdet(bh.h, C.byref(la), C.byref(sg)) < 0 and b"batched handle" in L.slu_b200_last_error()
    bh.close()
