"""Componentwise backward error of the GPU kernels, factorizations and solves (backward.py has the bounds): the diagonal
LU (one-CTA and 8-CTA cluster kernels), the panel TRSM in both cases, C - A B on both FP64 GEMM variants, in double and
doublecomplex, on dominant, non-dominant, graded, tiny-pivot, power-of-two-scaled and (complex) extreme-pivot inputs;
then every factorization route and the solves N / T / H on their factors.  test_backward_cpu.py shows the reference
meeting each bound on the same inputs, so a ratio over its bound here is a kernel defect, whatever the conditioning."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import backward as bw
from superlu_dist_b200 import capi, hostlib, matgen
from util import complex_problem, poisson_problem

pytestmark = pytest.mark.gpu
D, Z = np.float64, np.complex128


# --------------------------------------------------------------------------------------------------------- kernels
def diag_lu_case(family, ns, z):
    """-> (ratio, bound); the rows below the block are not the kernel's (the factorization's TRSM solves them)"""
    a = bw.diag_lu_input(family, ns, bw.vecs_for(ns, family) % 40, ns, z)
    out, info, tiny = capi.k_diag_lu(a, replace_tiny=1, thresh=bw.THRESH)
    r, rep = bw.diag_lu_ratio(a, out, bw.THRESH)
    assert info == 0 and rep == tiny, (info, rep, tiny)
    if family == "tiny":
        assert tiny == len([c for c in bw.TINY_COLS if c < ns])
    assert np.array_equal(out[ns:], a[ns:])
    return r, bw.kernel_bound(ns, a.dtype)


def trsm_l_case(family, ns, z):
    u, b = bw.trsm_l_input(family, ns, bw.vecs_for(ns, family), ns + 1, z)
    return bw.trsm_l_ratio(u, b, capi.k_trsm(u, b, ucase=False)), bw.kernel_bound(ns, u.dtype)


def trsm_u_case(family, ns, z):
    lo, b = bw.trsm_u_input(family, ns, bw.vecs_for(ns, family), ns + 2, z)
    return bw.trsm_u_ratio(lo, b, capi.k_trsm(lo, b, ucase=True)), bw.kernel_bound(ns, lo.dtype)


def gemm_case(family, shape, variant, z):
    m, n, k = shape
    a, b, c = bw.gemm_input(family, m, n, k, m + n + k, z)
    os.environ["SLU_B200_GEMM_VARIANT"] = str(variant)
    try:
        out, _ = capi.k_gemm_sub(a, b, c)
    finally:
        os.environ.pop("SLU_B200_GEMM_VARIANT", None)
    return bw.gemm_sub_ratio(a, b, c, out), bw.gemm_bound(k, c.dtype)


@pytest.mark.parametrize("z", [False, True], ids=["d", "z"])
@pytest.mark.parametrize("kernel", ["diag_lu", "trsm_l", "trsm_u"])
@pytest.mark.parametrize("family", bw.ZFAMILIES)
def test_kernel_backward_error(kernel, family, z):
    """Every width of the family (one parameter set per kernel, family and type: the widths run in one loop)"""
    if family == "zpivots" and not z:
        pytest.skip("complex pivots are a doublecomplex family")
    if kernel == "trsm_u" and family in ("tiny", "zpivots"):
        pytest.skip("a unit lower triangle has no pivots")
    fn = {"diag_lu": diag_lu_case, "trsm_l": trsm_l_case, "trsm_u": trsm_u_case}[kernel]
    bad = []
    for ns in (bw.ZWIDTHS if z else bw.WIDTHS):
        r, bound = fn(family, ns, z)
        if not r <= bound:
            bad.append((ns, r, bound))
    assert not bad, bad


@pytest.mark.parametrize("variant", [0, 30])
@pytest.mark.parametrize("family", bw.GEMM_FAMILIES)
def test_gemm_sub_backward_error(family, variant):
    results = [(s, *gemm_case(family, s, variant, False)) for s in bw.GEMM_SHAPES]
    assert all(r <= b for _, r, b in results), results


@pytest.mark.parametrize("family", bw.GEMM_FAMILIES)
def test_z_gemm_sub_backward_error(family):
    results = [(s, *gemm_case(family, s, 0, True)) for s in bw.GEMM_SHAPES]
    assert all(r <= b for _, r, b in results), results


# ---------------------------------------------------------------------------------------------- factorizations
NRHS = [1, 2, 17, 33]


def check_factors(prob, F, tiny=0, thresh=None, solve=None):
    """The factorization bound on layer 0 of prob (downloaded), replaced pivots counted; then, when `solve` is given
    (b, trans) -> x, the solve bound for every nrhs and trans on the same factors.  -> the largest ratio / bound"""
    L, U = bw.factors(prob, prob.layers[0])
    r, rep = bw.factor_ratio(F, L, U, thresh)
    bound = bw.factor_bound(prob)
    assert rep == tiny, (rep, tiny)
    assert r <= bound, (r, bound)
    worst = r / bound
    if solve is not None:
        rng = np.random.default_rng(prob.n)
        for nrhs in NRHS:
            for trans in "NTH":
                b = rng.standard_normal((nrhs, prob.n))
                if np.dtype(prob.dtype).kind == "c":
                    b = b + 1j * rng.standard_normal((nrhs, prob.n))
                rs = bw.solve_ratio(L, U, solve(b, trans), b, trans)
                assert rs <= bound, (nrhs, trans, rs, bound)
                worst = max(worst, rs / bound)
    return worst


def _problem(name):
    if name in bw.ZPROBLEMS:
        return complex_problem(**bw.ZPROBLEMS[name])
    return poisson_problem(**bw.PROBLEMS[name])[0]


@pytest.mark.parametrize("lookahead", [True, False], ids=["lookahead", "no_lookahead"])
@pytest.mark.parametrize("name", list(bw.PROBLEMS) + list(bw.ZPROBLEMS))
def test_pgstrf3d(name, lookahead):
    """pdgstrf3d_b200 / pzgstrf3d_b200 with the int8 path off"""
    prob = _problem(name)
    F = bw.panel_matrix(prob, prob.layers[0])
    fn = capi.pzgstrf3d if name in bw.ZPROBLEMS else capi.pdgstrf3d
    info, st = fn(prob, 0, tc_slices=-1, no_lookahead=0 if lookahead else 1)
    assert info == 0
    check_factors(prob, F, st.tiny_pivots)


def _handle_route(prob, F, fill):
    h = capi.Handle(prob, 0, tc_slices=-1)
    fill(h)
    assert h.factor() == 0
    h.download()
    try:
        return check_factors(prob, F, h.stats().tiny_pivots, solve=h.solve)
    finally:
        h.close()


@pytest.mark.parametrize("name", list(bw.PROBLEMS) + list(bw.ZPROBLEMS))
def test_handle_fill_csr_factor_solve(name):
    if name in bw.ZPROBLEMS:
        prob = complex_problem(**bw.ZPROBLEMS[name])
        _handle_route(prob, bw.panel_matrix(prob, prob.layers[0]), lambda h: h.upload())
        return
    prob, (rp, ci, v) = poisson_problem(**bw.PROBLEMS[name])
    vals = matgen.batch_values(rp, ci, v, 1, 5)[0]
    F = bw.csr_values(rp, ci, vals, prob.perm, prob.n)
    _handle_route(prob, F, lambda h: h.fill_csr(rp, ci, vals, prob.perm))


def test_indefinite_shift():
    from test_inertia_cpu import shifted
    prob, (rp, ci, v) = poisson_problem(**bw.SHIFT_KW)
    vals = shifted(rp, ci, v, bw.shift_sigma())
    F = bw.csr_values(rp, ci, vals, prob.perm, prob.n)
    _handle_route(prob, F, lambda h: h.fill_csr(rp, ci, vals, prob.perm))
    d = bw.factors(prob, prob.layers[0])[1].diagonal()
    assert (d < 0).any() and (d > 0).any()


@pytest.mark.parametrize("name", ["top256", "z32"])
def test_batched_members(name):
    from test_gpu_solve_complex import complex_csr
    kw = {**bw.PROBLEMS, **bw.ZPROBLEMS}[name]
    prob, rv = poisson_problem(**kw)
    cx = name in bw.ZPROBLEMS
    rp, ci, v = complex_csr(**kw) if cx else rv
    if cx:
        prob.dtype = np.dtype(np.complex128)
        lay = prob.layers[0]
        lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    vals = matgen.batch_values(rp, ci, v, 3, 1)
    h = capi.BatchHandle(prob, 3, tc_slices=-1)
    h.fill_csr(rp, ci, vals, prob.perm)
    assert not h.factor().any()
    rng = np.random.default_rng(3)
    for nrhs in NRHS:
        for trans in "NTH":
            b = rng.standard_normal((3, nrhs, prob.n)) + (1j * rng.standard_normal((3, nrhs, prob.n)) if cx else 0)
            x = h.solve(b, trans)
            for j in range(3):
                h.download(j)
                L, U = bw.factors(prob, prob.layers[0])
                assert bw.solve_ratio(L, U, x[j], b[j], trans) <= bw.factor_bound(prob), (j, nrhs, trans)
    for j in range(3):
        h.download(j)
        check_factors(prob, bw.csr_values(rp, ci, vals[j], prob.perm, prob.n))
    h.close()


def test_fill_csr_scaled_kkt_replaced_pivots():
    """Static pivoting: the matched, scaled KKT matrix with pivots below KKT_THRESH replaced by +-KKT_THRESH"""
    from test_gpu_static_pivot import problem
    from test_static_pivot_cpu import scale_values
    prob, rp, ci, v, perm_r = problem(bw.kkt_matrix())
    prob.replace_tiny_pivot, prob.thresh = 1, bw.KKT_THRESH
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs, equil=False)
    pr, R2, C2 = h.scaling()
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    F = bw.csr_values(rp, ci, scale_values(v, rows, ci, R2, C2), prob.perm, prob.n, pr)
    assert h.factor() == 0
    h.download()
    tiny = h.stats().tiny_pivots
    assert tiny > 0
    check_factors(prob, F, tiny, bw.KKT_THRESH, solve=h.solve)
    h.close()


@pytest.mark.parametrize("dtype", [D, Z], ids=["d", "z"])
def test_schur_handle(dtype):
    """A - [L11 0; L21 I] [U11 U12; 0 S] with S from schur(), on the 256-column top separator of Poisson 16^3"""
    from test_gpu_schur import make
    prob, (rp, ci, vals), s, _ = make("p16_w256", dtype, dense=False)
    h = capi.SchurHandle(prob, s, tc_slices=-1)
    h.fill_csr(rp, ci, vals, prob.perm)
    assert h.factor() == 0
    h.download()
    S = h.schur()
    h.close()
    n1 = prob.n - s
    L, U = bw.factors(prob, prob.layers[0], n_elim=n1)
    Sc = sp.coo_matrix(S)
    U = (U + sp.csr_matrix((Sc.data, (Sc.row + n1, Sc.col + n1)), shape=U.shape)).tocsr()
    F = bw.csr_values(rp, ci, vals, prob.perm, prob.n)
    r, _ = bw.factor_ratio(F, L, U)
    assert r <= bw.factor_bound(prob), r
