"""Static pivoting on the device routes: slu_b200_fill_csr_scaled, _get_scaling, _solve_scaled, their batched and
doublecomplex twins.  Matrices with a zero or dominated diagonal go through matching (sluh_large_diag_perm) -> ordering
of the row-permuted pattern -> symbolic -> scaled fill with device equilibration -> factor -> solve in A's own ordering,
checked against SciPy; the fill against the plain fill of the host-built Pr Dr A Dc, the equilibration against the NumPy
restatement of dgsequ / dlaqgs bit for bit."""
import numpy as np
import pytest
import scipy.sparse as sp

from superlu_dist_b200 import LUProblem, capi, hostlib
from test_static_pivot_cpu import csr_parts, equilibrate, example, kkt, poisson2d, scale_values

pytestmark = pytest.mark.gpu
RES_TOL = 1e-13


def problem(A, leaf=16, relax=8, maxsup=32, perm_r=None, nschur=0):
    """(LUProblem on the pattern of Pr A, with the values of Pr A in layer 0, rowptr, colind, values of A, perm_r)"""
    rp, ci, v = csr_parts(A)
    if perm_r is None:
        perm_r = hostlib.large_diag_perm(rp, ci, v)[0]
    prp, pci, pv = hostlib.row_permute(rp, ci, v, perm_r)
    perm = hostlib.nd_order_graph(prp, pci, leaf=leaf)
    prob = LUProblem.from_matrix(prp, pci, np.abs(pv), perm, relax=relax, maxsup=maxsup, nschur=nschur)
    if np.iscomplexobj(v):
        prob.dtype = np.dtype(np.complex128)
        for lay in prob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    return prob, rp, ci, v, perm_r


def arena(prob):
    lay = prob.layers[0]
    return lay.lval.copy(), lay.uval.copy()


def residual(A, x, b):
    """||A x - b|| / (||A|| ||x|| + ||b||) in the infinity norm, per right-hand side (rows)"""
    An = abs(A).sum(axis=1).max()
    return max(np.abs(A @ xj - bj).max() / (An * np.abs(xj).max() + np.abs(bj).max()) for xj, bj in zip(np.atleast_2d(x), np.atleast_2d(b)))


def op(A, trans):
    return {"N": A, "T": A.T, "H": A.conj().T}[trans].tocsr()


def complex_kkt(g, m, seed):
    A = kkt(g, m, seed)
    rng = np.random.default_rng(seed)
    return sp.csr_matrix((A.data * np.exp(0.3j * rng.standard_normal(A.nnz)), A.indices, A.indptr), shape=A.shape)


MATRICES = {"kkt": lambda tmp: kkt(16, 40, 3), "zkkt": lambda tmp: complex_kkt(12, 30, 4),
            "g4": lambda tmp: example("g4.rua", tmp), "g20": lambda tmp: example("g20.rua", tmp),
            "big": lambda tmp: example("big.rua", tmp), "cg20": lambda tmp: example("cg20.cua", tmp)}


@pytest.mark.parametrize("equil", [False, True])
@pytest.mark.parametrize("name", ["kkt", "zkkt", "big", "cg20"])
def test_fill_matches_the_plain_fill_of_the_host_scaled_matrix(tmp_path, name, equil):
    A = MATRICES[name](tmp_path)
    prob, rp, ci, v, perm_r = problem(A)
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    h = capi.Handle(prob, 0)
    out = h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs, equil=equil)
    pr2, R2, C2 = h.scaling()
    assert np.array_equal(pr2, perm_r)
    if equil:
        Re, Ce, rowcnd, colcnd, amax, equed = equilibrate(rp, ci, v, R, Cs)
        assert np.array_equal(R2, Re) and np.array_equal(C2, Ce)
        assert (out["rowcnd"], out["colcnd"], out["amax"], out["equed"]) == (rowcnd, colcnd, amax, equed)
    else:
        assert np.array_equal(R2, R) and np.array_equal(C2, Cs) and out["equed"] == 0
    h.download()
    mine = arena(prob)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    sv = scale_values(v, rows, ci, R2, C2)
    h.fill_csr(*hostlib.row_permute(rp, ci, sv, perm_r), prob.perm)
    h.download()
    ref = arena(prob)
    h.close()
    assert np.array_equal(mine[0], ref[0]) and np.array_equal(mine[1], ref[1])
    F = abs(sp.csr_matrix((sv, (rows, ci)), shape=A.shape))
    assert abs(out["max_abs"] - F.max()) <= 4 * np.finfo(np.float64).eps * F.max()   # the modulus: hypot on both sides
    assert abs(out["norm_inf"] - F.sum(axis=1).max()) <= 1e-14 * out["norm_inf"]


@pytest.mark.parametrize("name", list(MATRICES))
def test_solves_in_the_original_ordering(tmp_path, name):
    A = MATRICES[name](tmp_path)
    prob, rp, ci, v, perm_r = problem(A)
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    h = capi.Handle(prob, 0)
    out = h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs)
    assert h.factor() == 0
    rng = np.random.default_rng(7)
    dt = np.complex128 if np.iscomplexobj(v) else np.float64
    b = rng.standard_normal((2, A.shape[0])).astype(dt)
    if dt == np.complex128:
        b = b + 1j * rng.standard_normal(b.shape)
    for trans in ("N", "T", "H"):
        x = h.solve_scaled(b, trans=trans)
        assert residual(op(A, trans), x, b) <= RES_TOL, (name, trans)
        assert h.stats().reserved[5] > 0
    x1 = h.solve_scaled(b[0])
    assert residual(A, x1, b[0]) <= RES_TOL
    assert 0 < h.rcond(out["norm_inf"], "I") <= 1
    h.close()


def test_kkt_fails_through_the_plain_fill():
    """the zero block's unknowns ordered before their Poisson neighbours: exact zero pivots without the row permutation"""
    A = kkt(16, 40, 3)
    rp, ci, v = csr_parts(A)
    perm = np.concatenate([np.arange(256) + 40, np.arange(40)]).astype(np.int32)
    prob = LUProblem.from_matrix(rp, ci, v, perm, relax=8, maxsup=32)
    h = capi.Handle(prob, 0)
    h.fill_csr(rp, ci, v, prob.perm)
    assert h.factor() > 0
    h.close()


def test_equilibration_undoes_row_scaling():
    A = poisson2d(20)
    rng = np.random.default_rng(2)
    A = sp.csr_matrix(sp.diags(np.exp2(rng.choice([-30.0, 30.0], A.shape[0]))) @ A)
    prob, rp, ci, v, perm_r = problem(A, perm_r=np.arange(A.shape[0], dtype=np.int32))
    h = capi.Handle(prob, 0)
    out = h.fill_csr_scaled(rp, ci, v, prob.perm)
    assert out["rowcnd"] < 1e-15 and out["equed"] in (1, 3)
    _, R, Cs = h.scaling()
    again = h.fill_csr_scaled(rp, ci, v, prob.perm, None, R, Cs)
    assert again["rowcnd"] > 0.1 and again["equed"] == 0
    assert h.factor() == 0
    b = rng.standard_normal(A.shape[0])
    assert residual(A, h.solve_scaled(b), b) <= RES_TOL
    h.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_batched_family_shares_the_row_permutation(cplx):
    B = 8
    members = [kkt(14, 35, 9, sigma=0.01 * j) for j in range(B)]
    if cplx:
        members = [sp.csr_matrix(M * (1.0 + 0.2j)) for M in members]
    prob, rp, ci, v0, perm_r = problem(members[0])
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v0)
    vals = np.stack([csr_parts(M)[2] for M in members])
    assert all(np.array_equal(csr_parts(M)[1], ci) for M in members)
    bh = capi.BatchHandle(prob, B)
    out = bh.fill_csr_scaled(rp, ci, vals, prob.perm, perm_r, R, Cs)
    assert (bh.factor() == 0).all()
    rng = np.random.default_rng(3)
    b = rng.standard_normal((B, 2, prob.n)) * (1.0 + 0.5j if cplx else 1.0)
    x = bh.solve_scaled(b)
    launches = bh.stats().reserved[5]
    xt = bh.solve_scaled(b, trans="H")
    h = capi.Handle(prob, 0)
    for j, M in enumerate(members):
        o = h.fill_csr_scaled(rp, ci, vals[j], prob.perm, perm_r, R, Cs)
        Rj, Cj = bh.scaling(j)
        _, Ru, Cu = h.scaling()
        assert np.array_equal(Rj, Ru) and np.array_equal(Cj, Cu)
        assert all(out[k][j] == o[k] for k in ("rowcnd", "colcnd", "amax", "equed", "max_abs"))
        assert residual(M, x[j], b[j]) <= RES_TOL
        assert residual(op(M, "H"), xt[j], b[j]) <= RES_TOL
    assert h.factor() == 0
    h.solve_scaled(b[-1])
    assert h.stats().reserved[5] == launches
    per = np.stack([R * (1.0 + 0.01 * j) for j in range(B)])
    bh.fill_csr_scaled(rp, ci, vals, prob.perm, perm_r, per, np.stack([Cs] * B), equil=False)
    assert np.array_equal(bh.scaling(5)[0], per[5])
    h.close()
    bh.close()


def test_refusals_leave_the_handle_usable():
    A = kkt(10, 20, 5)
    prob, rp, ci, v, perm_r = problem(A)
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    h = capi.Handle(prob, 0)
    b = np.random.default_rng(0).standard_normal(A.shape[0])
    with pytest.raises(RuntimeError, match="scaled fill"):
        h.solve_scaled(b)
    with pytest.raises(RuntimeError, match="scaled fill"):
        h.scaling()
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs)
    assert h.factor() == 0
    bad_perm = perm_r.copy()
    bad_perm[0] = bad_perm[1]
    for kw, msg in ((dict(perm_r=bad_perm), "perm_r is not a permutation"), (dict(R=np.where(np.arange(len(R)) == 3, 0.0, R)), "R\\[3\\]"),
                    (dict(C=np.where(np.arange(len(R)) == 2, np.nan, Cs)), "C\\[2\\]")):
        args = dict(perm_r=perm_r, R=R, C=Cs)
        args.update(kw)
        with pytest.raises(RuntimeError, match=msg):
            h.fill_csr_scaled(rp, ci, v, prob.perm, **args)
    with pytest.raises(RuntimeError, match="perm is not a permutation"):
        h.fill_csr_scaled(rp, ci, v, np.zeros_like(prob.perm), perm_r, R, Cs)
    with pytest.raises(RuntimeError, match="row 4 of A is exactly zero"):
        h.fill_csr_scaled(rp, ci, np.where(np.repeat(np.arange(len(rp) - 1), np.diff(rp)) == 4, 0.0, v), prob.perm, perm_r, R, Cs)
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs)
    assert h.factor() == 0
    assert residual(A, h.solve_scaled(b), b) <= RES_TOL
    # a later plain fill or upload drops the scaling
    prp, pci, pv = hostlib.row_permute(rp, ci, v, perm_r)
    h.fill_csr(prp, pci, pv, prob.perm)
    assert h.factor() == 0
    with pytest.raises(RuntimeError, match="scaled fill"):
        h.solve_scaled(b)
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs)
    h.upload()
    with pytest.raises(RuntimeError, match="scaled fill"):
        h.solve_scaled(b)
    h.close()
    # batched: a plain batch_fill_csr or batch_fill_affine drops it too
    bh = capi.BatchHandle(prob, 2)
    vals = np.stack([v, 2.0 * v])
    for refill in (lambda: bh.fill_csr(prp, pci, np.stack([pv, 2.0 * pv]), prob.perm),
                   lambda: bh.fill_affine(prp, pci, pv[None], np.ones((2, 1)), prob.perm)):
        bh.fill_csr_scaled(rp, ci, vals, prob.perm, perm_r, R, Cs)
        refill()
        bh.factor()
        with pytest.raises(RuntimeError, match="scaled fill"):
            bh.solve_scaled(np.stack([b, b]))
    with pytest.raises(RuntimeError, match="batched handle"):
        capi.Handle.fill_csr_scaled(bh, rp, ci, v, prob.perm, perm_r, R, Cs)
    bh.close()
    # Schur handles
    sperm = hostlib.schur_order(prp, pci, np.arange(A.shape[0] - 8, A.shape[0]))
    sprob = LUProblem.from_matrix(prp, pci, np.abs(pv), sperm, relax=8, maxsup=32, nschur=8)
    sh = capi.SchurHandle(sprob, 8)
    with pytest.raises(RuntimeError, match="Schur handle"):
        sh.fill_csr_scaled(rp, ci, v, sprob.perm, perm_r, R, Cs)
    sh.close()
