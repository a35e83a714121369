"""Every single-GPU route on unsymmetric patterns stored as exact skylines (LUProblem.prune_u; the cases and their host
counts are in test_unsym_skyline_cpu.py): short U segments on wide supernodes and on the big Schur tiles, dropped
columns and blocks, and more than one staging round of the skyline <-> dense-packed U conversion.

Bars: the factors against the oracle at rel_err < 1e-10 per arena (the other parity tests' bar); solves against SciPy
on F = P A P^T; rcond against the LAPACK-checked restatement; selected inversion against a dense inverse (small cases)
or oracle/selinv.py run on the GPU's own factors."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle, selinv
from superlu_dist_b200 import capi
from test_gpu_gscon import check_estimate
from test_gpu_selinv import csr_of, stored_positions
from test_gpu_solve_trans import check_against_scipy, permuted
from test_selinv_complex_cpu import complex_logdet
from test_unsym_skyline_cpu import LARGE, SMALL, counts, l_rows, make, pattern, u_columns, values
from util import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10


@functools.lru_cache(maxsize=8)
def _oracle(name, complex_, seed=0):
    """-> (lval, uval, ops_fact) of the oracle on the pruned problem"""
    prob = make(name, values(name, complex_, seed))
    info, ops, _ = oracle.factor(prob)
    assert info == 0
    return prob.layers[0].lval, prob.layers[0].uval, ops


def _check(prob, name, complex_, seed=0, tol=TOL):
    rl, ru, _ = _oracle(name, complex_, seed)
    lay = prob.layers[0]
    el, eu = rel_err(lay.lval, rl), rel_err(lay.uval, ru)
    assert el < tol and eu < tol, (name, el, eu)


def _factored(name, complex_=False, seed=0, **opt):
    prob = make(name, values(name, complex_, seed))
    h = capi.Handle(prob, 0, **opt)
    h.upload()
    assert h.factor() == 0
    h.download()
    return prob, h


def _f(name, complex_=False, seed=0):
    rp, ci, _, perm = pattern(name)
    return permuted(rp, ci, values(name, complex_, seed), perm)


ROUTES = [pytest.param(name, c, opt, id=f"{name}-{tag}") for name in SMALL + LARGE
          for c, opt, tag in ((False, {}, "double"), (False, dict(tc_slices=-1), "double_fp64"), (True, {}, "complex"))]


@pytest.mark.parametrize("name,complex_,opt", ROUTES)
def test_handle_matches_oracle(name, complex_, opt):
    """upload / factor / download against the oracle; the operation count against the oracle's, and nnz_u against
    sum ns * ncols from the index arrays.  The band case needs three staging rounds of the U conversion both ways."""
    prob, h = _factored(name, complex_, **opt)
    st = h.stats()
    h.close()
    _check(prob, name, complex_)
    ops = _oracle(name, complex_)[2]
    assert abs(st.ops_fact - ops) <= 1e-9 * ops, (st.ops_fact, ops)
    c = counts(name)
    assert st.nnz_u == c["nnz_u"]
    if name == "band":
        assert c["staging_rounds"] >= 2


@pytest.mark.parametrize("name", ["band", "upwind"])
def test_lookahead_on_off_agree(name):
    a, h = _factored(name)
    h.close()
    b, h = _factored(name, no_lookahead=1)
    h.close()
    for x, y in ((a.layers[0].lval, b.layers[0].lval), (a.layers[0].uval, b.layers[0].uval)):
        assert rel_err(x, y) < 1e-12


@pytest.mark.parametrize("name", ["band_small", "upwind_small", "band", "upwind_fem"])
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_fill_csr_equals_upload(name, complex_):
    """fill_csr puts exactly the values the host fill does (host arrays poisoned first); factors from it match the
    oracle."""
    vals = values(name, complex_)
    prob = make(name, vals)
    want = prob.layers[0].copy()
    prob.layers[0].lval[:] = -7.0
    prob.layers[0].uval[:] = -7.0
    rp, ci, _, perm = pattern(name)
    h = capi.Handle(prob, 0)
    h.fill_csr(rp, ci, vals, perm)
    h.download()
    assert np.array_equal(prob.layers[0].lval, want.lval) and np.array_equal(prob.layers[0].uval, want.uval)
    assert h.factor() == 0
    h.download()
    h.close()
    _check(prob, name, complex_)


@pytest.mark.parametrize("name", ["upwind_small", "band", "upwind"])
def test_factor_host_and_overlapped_drop_in(name):
    """factor_host and pdgstrf3d_b200 with the overlapped transfers fall back to the plain path on short skylines: the
    same factors as upload / factor / download."""
    ref, h = _factored(name)
    h.close()
    p1 = make(name, values(name))
    h = capi.Handle(p1, 0)
    assert h.factor_host() == 0
    h.close()
    p2 = make(name, values(name))
    h = capi.Handle(p2, 0, overlap_h2d=1)
    assert h.factor_host() == 0
    h.close()
    p3 = make(name, values(name))
    info, _ = capi.pdgstrf3d(p3, 0, pipeline=1, overlap_h2d=1)
    assert info == 0
    for p in (p1, p2, p3):
        assert rel_err(p.layers[0].lval, ref.layers[0].lval) < 1e-12
        assert rel_err(p.layers[0].uval, ref.layers[0].uval) < 1e-12


@pytest.mark.parametrize("name", ["band_small", "band"])
def test_refactor_equals_fresh_handle(name):
    """Refactoring one handle with new values, through upload and through fill_csr, equals a fresh handle: nothing of
    the previous factors survives in the dense-packed padding."""
    rp, ci, _, perm = pattern(name)
    prob = make(name, values(name, seed=0))
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    other = make(name, values(name, seed=1))
    prob.layers[0].lval[:] = other.layers[0].lval
    prob.layers[0].uval[:] = other.layers[0].uval
    h.upload()
    assert h.factor() == 0
    h.download()
    _check(prob, name, False, seed=1)
    h.fill_csr(rp, ci, values(name, seed=0), perm)
    assert h.factor() == 0
    h.download()
    h.close()
    _check(prob, name, False, seed=0)


@pytest.mark.parametrize("name", ["upwind_small", "upwind_fem"])
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_batched_members(name, complex_):
    """BatchHandle, B = 3: each member's factors against the oracle, batched solves N and T against SciPy."""
    B = 3
    rp, ci, _, perm = pattern(name)
    vals = [values(name, complex_, seed=s) for s in range(B)]
    prob = make(name, vals[0])
    bh = capi.BatchHandle(prob, B)
    bh.fill_csr(rp, ci, np.stack(vals), perm)
    assert not bh.factor().any()
    for j in range(B):
        bh.download(j)
        _check(prob, name, complex_, seed=j)
    rng = np.random.default_rng(4)
    b = rng.standard_normal((B, 2, prob.n))
    if complex_:
        b = b + 1j * rng.standard_normal(b.shape)
    for trans in ("N", "T"):
        x = bh.solve(b, trans=trans)
        for j in range(B):
            check_against_scipy(_f(name, complex_, seed=j), trans, b[j], x[j])
    bh.close()


@pytest.mark.parametrize("name", ["band_small", "upwind_small", "upwind_fem_small", "band"])
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_solves(name, complex_):
    prob, h = _factored(name, complex_)
    F = _f(name, complex_)
    rng = np.random.default_rng(5)
    b = rng.standard_normal((3, prob.n))
    if complex_:
        b = b + 1j * rng.standard_normal(b.shape)
    for trans in ("N", "T", "H"):
        for rhs in (b, b[0]):
            x = h.solve(rhs, trans=trans)
            check_against_scipy(F, trans, rhs, x)
    h.close()


@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_rcond(name, complex_):
    prob, h = _factored(name, complex_)
    F = _f(name, complex_)
    for norm in ("1", "I"):
        check_estimate(h, F, norm)
    h.close()


def _no_slot(prob, r, c):
    """How many positions (r, c) of the factored ordering have no slot for selinv_get: not in an L panel's rows, nor
    in a stored column of a U panel (the dense-packed rows above the skyline start count as slots)."""
    xsup = np.asarray(prob.xsup)
    sup = np.searchsorted(xsup, np.arange(prob.n), side="right") - 1
    lset, uc = {}, u_columns(prob)
    bad = 0
    for i, j in zip(r.tolist(), c.tolist()):
        if i >= xsup[sup[j]]:
            s = sup[j]
            if s not in lset:
                lset[s] = set(l_rows(prob, s).tolist())
            bad += i not in lset[s]
        else:
            k = sup[i]
            bad += k not in uc or j not in set(uc[k][0].tolist())
    return bad


@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_selinv_small_against_dense_inverse(name, complex_):
    """On the pattern of A^T every entry of A^-1 comes back and equals the dense inverse; on the pattern of A the call
    fails with the host-computed count of entries without a slot; the entries of H in the dense-packed padding (rows
    of a stored U column above its skyline start) equal the dense inverse too; logdet against slogdet."""
    prob, h = _factored(name, complex_)
    rp, ci, _, perm = pattern(name)
    n = prob.n
    vals = values(name, complex_)
    A = np.zeros((n, n), vals.dtype)
    rows = np.repeat(np.arange(n), np.diff(rp))
    A[rows, ci] = vals
    G = np.linalg.inv(A)
    h.selinv()
    # pattern of A^T: entries (ci[p], rows[p])
    trp, tci, order = csr_of(ci.astype(np.int64), rows.astype(np.int64), n)
    got = h.inv_entries(trp, tci, perm)
    ref = G[ci[order], rows[order]]
    assert np.abs(got - ref).max() <= TOL * np.abs(ref).max()
    # pattern of A: A^-1(i, j) sits at H(perm j, perm i)
    want = _no_slot(prob, np.asarray(perm)[ci], np.asarray(perm)[rows])
    assert want > 0
    with pytest.raises(RuntimeError, match=f"selinv_get: {want} entries have no slot"):
        h.inv_entries(rp, ci, perm)
    # the padding: H(r, c) for r in [f, fstnz) of every stored column c of U panel k, i.e. A^-1(iperm c, iperm r)
    xsup = np.asarray(prob.xsup)
    pr, pc = [], []
    for k, (cols, fst) in u_columns(prob).items():
        for c, f in zip(cols.tolist(), fst.tolist()):
            pr += range(int(xsup[k]), f)
            pc += [c] * (f - int(xsup[k]))
    assert len(pr) > 0
    iperm = np.argsort(perm)
    ai, aj = iperm[np.array(pc)], iperm[np.array(pr)]
    prp, pci, order = csr_of(ai, aj, n)
    got = h.inv_entries(prp, pci, perm)
    ref = G[ai[order], aj[order]]
    assert np.abs(got - ref).max() <= TOL * np.abs(G).max()
    sign, logabs = h.logdet()
    s2, l2 = np.linalg.slogdet(A)
    assert abs(sign - s2) <= 1e-12 and abs(logabs - l2) <= 1e-12 * max(1.0, abs(l2))
    h.close()


@pytest.mark.parametrize("name", ["upwind", "upwind_fem", "band"])
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_selinv_against_oracle(name, complex_):
    prob, h = _factored(name, complex_)
    lay = prob.layers[0]
    h.selinv()
    hl, hu = selinv.selinv(prob, lay)
    rows, cols, u = stored_positions(prob, lay)
    rp, ci, order = csr_of(cols, rows, prob.n)
    got = np.empty(len(rows), hl.dtype)
    got[order] = h.inv_entries(rp, ci, np.arange(prob.n, dtype=np.int32))
    ref = np.concatenate([hl, hu[u]])
    assert np.abs(got - ref).max() <= TOL * np.abs(ref).max()
    sign, logabs = h.logdet()
    s2, l2 = (complex_logdet if complex_ else selinv.logdet)(prob, lay)
    assert abs(sign - s2) <= 1e-12 and abs(logabs - l2) <= 1e-12 * abs(l2)
    h.close()


@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_fill_csr_refuses_entry_above_skyline(complex_):
    """One extra entry of A above its U column's skyline start: fill_csr fails and counts exactly that entry."""
    name = "band_small"
    prob = make(name)
    rp, ci, _, perm = pattern(name)
    k, (cols, fst) = next((k, c) for k, c in u_columns(prob).items() if (c[1] > prob.xsup[k]).any())
    q = int(np.nonzero(fst > prob.xsup[k])[0][0])
    iperm = np.argsort(perm)
    i, j = int(iperm[prob.xsup[k]]), int(iperm[cols[q]])
    rows = np.append(np.repeat(np.arange(prob.n), np.diff(rp)), i)
    cis = np.append(ci, j)
    vals = np.append(values(name, complex_), 1.0)
    a = sp.csr_matrix((vals, (rows, cis)), shape=(prob.n, prob.n))
    a.sort_indices()
    assert a.nnz == len(ci) + 1
    fill_prob = make(name, values(name, complex_))
    h = capi.Handle(fill_prob, 0)
    with pytest.raises(RuntimeError, match=r"(^|\D)1 entries of A have no slot"):
        h.fill_csr(a.indptr, a.indices, a.data, perm)
    h.close()
