"""The slot and scaling conventions of the gradient calls on the CPU oracle (superlu_dist_b200.autograd,
slu_b200_logdet_grad_device, slu_b200_solve_grad_device), without a GPU.  A scaled fill stores F = Pr Dr A Dc (factored as
Pc F Pc^T); selected inversion gives H = (Pc F Pc^T)^-T, so entry (i, j) of A reads H at (perm[perm_r[i]], perm[j]), and
R_i C_j H(perm[perm_r[i]], perm[j]) = A^-T(i, j): the gradient of log |det A| (its conjugate A^-H in complex).  The solve's
gradient -lambda x^T on the pattern, lambda = A^-T dL/dx, is checked against central differences."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle, selinv
from superlu_dist_b200 import LUProblem, hostlib
from test_static_pivot_cpu import csr_parts, kkt


def matrix(cplx):
    A = sp.csr_matrix(kkt(10, 24, 3))
    if cplx:
        rng = np.random.default_rng(4)
        A = sp.csr_matrix((A.data + 1j * 0.3 * rng.uniform(-1, 1, A.nnz), A.indices, A.indptr), shape=A.shape)
    return A


def scaled_factors(A):
    """(perm_r, R, C, perm, hl, hu, panels) of F = Pr Dr A Dc, factored by the oracle with its selected inverse; perm is the
    problem's final ordering (from_matrix may refine the one it is given)"""
    rp, ci, v = csr_parts(A)
    n = A.shape[0]
    perm_r, R, Cs, _ = hostlib.large_diag_perm(rp, ci, np.abs(v) if np.iscomplexobj(v) else v)
    rows = np.repeat(np.arange(n), np.diff(rp))
    F = sp.csr_matrix(((R[rows] * v) * Cs[ci], (perm_r[rows], ci)), shape=(n, n))
    F.sort_indices()
    frp, fci = F.indptr.astype(np.int32), F.indices.astype(np.int32)
    perm = hostlib.nd_order_graph(frp, fci, leaf=8)
    prob = LUProblem.from_matrix(frp, fci, F.data.real.copy(), perm, relax=8, maxsup=16)
    if np.iscomplexobj(v):
        im = LUProblem.from_matrix(frp, fci, F.data.imag.copy(), perm, relax=8, maxsup=16)
        prob.dtype = np.dtype(np.complex128)
        for z, lay in prob.layers.items():
            lay.lval = lay.lval.astype(np.complex128) + 1j * im.layers[z].lval
            lay.uval = lay.uval.astype(np.complex128) + 1j * im.layers[z].uval
    assert oracle.factor(prob)[0] == 0
    lay = prob.layers[0]
    hl, hu = selinv.selinv(prob, lay)
    return perm_r, R, Cs, np.asarray(prob.perm), hl, hu, selinv._Panels(prob, lay)


@pytest.mark.parametrize("cplx", [False, True])
def test_scaled_inverse_on_the_pattern_is_the_logdet_gradient(cplx):
    A = matrix(cplx)
    rp, ci, v = csr_parts(A)
    n = A.shape[0]
    perm_r, R, Cs, perm, hl, hu, P = scaled_factors(A)
    rows = np.repeat(np.arange(n), np.diff(rp))
    p, q = perm[perm_r[rows]], perm[ci]
    H = np.array([P.gather(hl, hu, np.array([a]), np.array([b]))[0, 0] for a, b in zip(p, q)])
    g = R[rows] * Cs[ci] * H
    Ainv = np.linalg.inv(A.toarray())
    ref = Ainv.T[rows, ci]
    tol = 1e-12 * np.linalg.cond(A.toarray()) * np.abs(ref).max()
    assert np.abs(g - ref).max() <= tol
    if cplx:
        assert np.abs(np.conj(g) - Ainv.conj().T[rows, ci]).max() <= tol
    # the gradient of log |det A| by central differences on a few entries
    _, l0 = np.linalg.slogdet(A.toarray())
    for e in np.random.default_rng(1).choice(len(v), 6, replace=False):
        h = 1e-6 * max(abs(v[e]), 1.0)
        Ap, Am = A.toarray(), A.toarray()
        Ap[rows[e], ci[e]] += h
        Am[rows[e], ci[e]] -= h
        fd = (np.linalg.slogdet(Ap)[1] - np.linalg.slogdet(Am)[1]) / (2 * h)
        assert abs(fd - g[e].real) <= 1e-6 * max(1.0, abs(g[e])), (e, fd, g[e])


def test_sampled_product_is_the_solve_gradient():
    A = matrix(False)
    rp, ci, v = csr_parts(A)
    n = A.shape[0]
    rows = np.repeat(np.arange(n), np.diff(rp))
    rng = np.random.default_rng(2)
    b, w = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))

    def loss(vals):
        return float((w * np.linalg.solve(sp.csr_matrix((vals, ci, rp), shape=(n, n)).toarray(), b)).sum())

    Ad = A.toarray()
    x = np.linalg.solve(Ad, b)
    lam = np.linalg.solve(Ad.T, w)
    g = -(lam[rows] * x[ci]).sum(axis=1)
    for e in rng.choice(len(v), 8, replace=False):
        h = 1e-6 * max(abs(v[e]), 1.0)
        vp, vm = v.copy(), v.copy()
        vp[e] += h
        vm[e] -= h
        fd = (loss(vp) - loss(vm)) / (2 * h)
        assert abs(fd - g[e]) <= 1e-6 * max(1.0, abs(g[e])), (e, fd, g[e])
