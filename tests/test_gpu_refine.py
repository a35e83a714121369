"""slu_b200_gsrfs and its batched / doublecomplex twins: iterative refinement with error bounds on the factors of a scaled
fill.  berr is checked bit for bit against the NumPy restatement of tests/test_refine_cpu.py evaluated on the returned x,
ferr against the same restatement's dlacn2 driven by SciPy solves, and the refined solutions against SciPy."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from superlu_dist_b200 import LUProblem, capi, hostlib
from test_gpu_static_pivot import MATRICES, RES_TOL, problem, residual
from test_gscon_cpu import lacn2
from test_refine_cpu import abs1, berr_of, ferr_weights, residual_rows
from test_static_pivot_cpu import csr_parts, kkt

pytestmark = pytest.mark.gpu
BERR_TOL = 1e-14
DENSE_MAX = 5000     # orders up to which the true forward error comes from a long-double refined reference


def prepared(A, equil=True):
    """a Handle after the scaled fill (matching and scalings from sluh_large_diag_perm) and a successful factor"""
    prob, rp, ci, v, perm_r = problem(A)
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs, equil=equil)
    assert h.factor() == 0
    return h, prob, rp, ci, v, perm_r, R, Cs


def rhs(shape, cplx, seed):
    rng = np.random.default_rng(seed)
    b = rng.standard_normal(shape)
    return b + 1j * rng.standard_normal(shape) if cplx else b


def numpy_berr(rp, ci, v, x, b):
    return berr_of(*residual_rows(rp, ci, v, x, b))


def check_columns(A, rp, ci, v, b, x, berr, steps, name=""):
    """property 1 (berr = the restatement on the returned x, bit for bit) and property 2 (berr <= 1e-14, the normwise
    residual bar of solve_scaled, 0 <= steps <= 20), per column"""
    for j in range(b.shape[0]):
        assert berr[j] == numpy_berr(rp, ci, v, x[j], b[j]), (name, j, berr[j], numpy_berr(rp, ci, v, x[j], b[j]))
        assert berr[j] <= BERR_TOL, (name, j, berr[j])
        if np.any(b[j]):      # a zero column stays exactly 0: no residual to normalise
            assert residual(A, x[j], b[j]) <= RES_TOL, (name, j)
        assert 0 <= steps[j] <= 20


@pytest.mark.parametrize("name", list(MATRICES))
def test_refines_solve_scaled(tmp_path, name):
    A = MATRICES[name](tmp_path)
    h, prob, rp, ci, v, *_ = prepared(A)
    b = rhs((2, A.shape[0]), np.iscomplexobj(v), 5)
    x0 = h.solve_scaled(b)
    x, berr, steps, ferr = h.refine(b, x0, ferr=False)
    assert ferr is None
    check_columns(A, rp, ci, v, b, x, berr, steps, name)
    print(f"\n{name}: n={A.shape[0]} berr {berr} steps {steps}")
    assert h.stats().reserved[5] > 0
    x1, berr1, steps1, _ = h.refine(b[0], x0[0], ferr=False)
    assert berr1 == numpy_berr(rp, ci, v, x1, b[0]) and berr1 <= BERR_TOL
    h.close()


def test_tiny_pivots_are_recovered():
    """KKT without the row permutation, the constraints eliminated first: every constraint's pivot is an exact zero,
    replaced by sqrt(eps) ||A|| (GESP).  solve_scaled's x carries the perturbation; refinement recovers full accuracy.
    Chosen on the CPU with the restatement on a dense unpivoted LU with the same replacements: 40 replaced pivots, berr
    1.4e-6 before, 3 steps to 1.5e-16."""
    A = kkt(16, 40, 3)
    n = A.shape[0]
    rp, ci, v = csr_parts(A)
    perm = np.concatenate([np.arange(256) + 40, np.arange(40)]).astype(np.int32)
    prob = LUProblem.from_matrix(rp, ci, v, perm, relax=8, maxsup=32)
    prob.replace_tiny_pivot = 1
    prob.thresh = np.sqrt(np.finfo(np.float64).eps) * abs(A).sum(axis=1).max()
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v, prob.perm, equil=False)
    assert h.factor() == 0
    assert h.stats().tiny_pivots > 0
    b = rhs(n, False, 1)
    x0 = h.solve_scaled(b)
    assert numpy_berr(rp, ci, v, x0, b) > 1e-10
    x, berr, steps, _ = h.refine(b, x0, ferr=False)
    assert steps >= 1 and berr <= BERR_TOL, (steps, berr)
    assert berr == numpy_berr(rp, ci, v, x, b)
    xs = spl.spsolve(A.tocsc(), b)
    before, after = np.abs(x0 - xs).max(), np.abs(x - xs).max()
    assert after * 100 <= before, (before, after)
    print(f"\ntiny pivots: {h.stats().tiny_pivots} replaced, berr {numpy_berr(rp, ci, v, x0, b):.2e} -> {berr:.2e} in {steps} steps, "
          f"forward error {before:.2e} -> {after:.2e}")
    h.close()


@pytest.mark.parametrize("name", ["kkt", "zkkt"])
def test_columns_are_independent(tmp_path, name):
    A = MATRICES[name](tmp_path)
    h, prob, rp, ci, v, *_ = prepared(A)
    cplx = np.iscomplexobj(v)
    n = A.shape[0]
    b = np.stack([np.zeros(n), rhs(n, cplx, 1), rhs(n, cplx, 2)]).astype(v.dtype)
    x0 = np.stack([np.zeros(n), np.zeros(n), h.solve_scaled(b[2])]).astype(v.dtype)
    x, berr, steps, _ = h.refine(b, x0, ferr=False)
    assert np.array_equal(x[0], np.zeros(n)) and berr[0] == 0.0 and steps[0] == 0
    assert steps[1] >= 1
    check_columns(A, rp, ci, v, b, x, berr, steps, name)
    for j in range(3):   # alone, each column ends within the same properties
        xj, bj, sj, _ = h.refine(b[j], x0[j], ferr=False)
        check_columns(A, rp, ci, v, b[j:j + 1], xj[None], [bj], [sj], name)
    h.close()


def true_forward_error(A, x, b):
    """||x - x*|| / ||x|| with x* from SciPy plus residual refinement in long double"""
    Ac = A.tocsc()
    ldt = np.clongdouble if np.iscomplexobj(A.data) or np.iscomplexobj(b) else np.longdouble
    data, idx, ptr = A.data.astype(ldt), A.indices, A.indptr
    xs = spl.spsolve(Ac, b)
    xl = xs.astype(ldt)
    for _ in range(3):
        r = b.astype(ldt) - np.add.reduceat(data * xl[idx], ptr[:-1])
        xl = xl + spl.spsolve(Ac, r.astype(b.dtype if np.iscomplexobj(b) else np.float64)).astype(ldt)
    return float(np.abs(x.astype(ldt) - xl).max() / np.abs(xl).max())


@pytest.mark.parametrize("name", list(MATRICES))
def test_forward_error_bound(tmp_path, name):
    A = MATRICES[name](tmp_path)
    h, prob, rp, ci, v, *_ = prepared(A)
    cplx = np.iscomplexobj(v)
    n = A.shape[0]
    b = rhs((2, n), cplx, 9)
    x, berr, steps, ferr = h.refine(b, h.solve_scaled(b))
    assert h.stats().reserved[5] > 0
    lu = spl.splu(A.tocsc())
    for j in range(2):
        assert berr[j] == numpy_berr(rp, ci, v, x[j], b[j])
        W = ferr_weights(*residual_rows(rp, ci, v, x[j], b[j]))
        est, _ = lacn2(lambda t: W * lu.solve(t, trans="H" if cplx else "T"), lambda t: lu.solve(W * t), n, cplx)
        ref = est / abs1(x[j]).max()
        assert abs(ferr[j] - ref) <= 1e-10 * ref, (name, j, ferr[j], ref)
        if n <= DENSE_MAX:
            true = true_forward_error(A, x[j], b[j])
            assert ferr[j] >= true, (name, j, ferr[j], true)
    print(f"\n{name}: ferr {ferr} berr {berr} steps {steps}")
    h.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_batched_members(cplx):
    B = 3
    members = [kkt(14, 35, 9, sigma=0.05 * j) for j in range(B)]
    if cplx:
        members = [sp.csr_matrix(M * (1.0 + 0.3j * (j + 1))) for j, M in enumerate(members)]
    prob, rp, ci, v0, perm_r = problem(members[0])
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v0)
    vals = np.stack([csr_parts(M)[2] for M in members])
    bh = capi.BatchHandle(prob, B)
    per = np.stack([R * (1.0 + 0.1 * j) for j in range(B)]), np.stack([Cs * (1.0 - 0.1 * j) for j in range(B)])
    bh.fill_csr_scaled(rp, ci, vals, prob.perm, perm_r, *per)
    assert (bh.factor() == 0).all()
    b = rhs((B, 2, prob.n), cplx, 4)
    x0 = bh.solve_scaled(b)
    x, berr, steps, ferr = bh.refine(b, x0)
    assert berr.shape == steps.shape == ferr.shape == (B, 2)
    for j, M in enumerate(members):
        check_columns(M, rp, ci, vals[j], b[j], x[j], berr[j], steps[j], f"member {j}")
        assert (ferr[j] > 0).all() and np.isfinite(ferr[j]).all()
    print(f"\nbatched ({'complex' if cplx else 'real'}): berr {berr.ravel()} steps {steps.ravel()}")
    # a member with an exact zero pivot is refused by name
    bad = vals.copy()
    bad[1] = 0.0
    bh.fill_csr_scaled(rp, ci, bad, prob.perm, perm_r, R, Cs, equil=False)
    info = bh.factor()
    assert info[1] > 0
    with pytest.raises(RuntimeError, match="member 1 has an exact zero pivot"):
        bh.refine(b, x0)
    bh.fill_csr_scaled(rp, ci, vals, prob.perm, perm_r, *per)
    assert (bh.factor() == 0).all()
    x2, berr2, _, _ = bh.refine(b, bh.solve_scaled(b), ferr=False)
    for j, M in enumerate(members):
        assert residual(M, x2[j], b[j]) <= RES_TOL and (berr2[j] <= BERR_TOL).all()
    bh.close()


def test_refusals_leave_the_handle_usable():
    A = kkt(10, 20, 5)
    prob, rp, ci, v, perm_r = problem(A)
    _, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    n = A.shape[0]
    b = rhs(n, False, 0)
    h = capi.Handle(prob, 0)

    def usable():
        h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs)
        assert h.factor() == 0
        x = h.solve_scaled(b)
        assert residual(A, x, b) <= RES_TOL
        return x

    with pytest.raises(RuntimeError, match="scaled fill"):
        h.refine(b, np.zeros(n))
    usable()
    # unfactored after the scaled fill
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, Cs)
    with pytest.raises(RuntimeError, match="successful slu_b200_factor after the scaled fill"):
        h.refine(b, np.zeros(n))
    x = usable()
    # a plain fill_csr after the scaled fill drops the kept A
    prp, pci, pv = hostlib.row_permute(rp, ci, v, perm_r)
    h.fill_csr(prp, pci, pv, prob.perm)
    assert h.factor() == 0
    with pytest.raises(RuntimeError, match="scaled fill"):
        h.refine(b, x)
    x = usable()
    # ldb, ldx, nrhs, null arguments through the C call
    fn = capi._fn("gsrfs", False)
    bb, xx, berr = b.copy(), x.copy(), np.zeros(1)
    for args, msg in (((n - 1, n, 1), "ldb"), ((n, n - 1, 1), "ldx"), ((n, n, 0), "nrhs")):
        assert fn(h.h, capi._ptr(bb), args[0], capi._ptr(xx), args[1], args[2], capi._ptr(berr), None, None) != 0
        assert msg in capi.lib().slu_b200_last_error().decode()
    assert fn(h.h, capi._ptr(bb), n, capi._ptr(xx), n, 1, None, None, None) != 0
    assert "null argument" in capi.lib().slu_b200_last_error().decode()
    assert np.array_equal(xx, x)
    x = usable()
    xr, br, sr, _ = h.refine(b, x)
    assert br <= BERR_TOL
    h.close()
    # batched: a plain batch_fill_csr drops the kept A
    bh = capi.BatchHandle(prob, 2)
    vals = np.stack([v, 2.0 * v])
    bh.fill_csr_scaled(rp, ci, vals, prob.perm, perm_r, R, Cs)
    bh.fill_csr(prp, pci, np.stack([pv, 2.0 * pv]), prob.perm)
    bh.factor()
    with pytest.raises(RuntimeError, match="scaled fill"):
        bh.refine(np.stack([b, b]), np.zeros((2, n)))
    with pytest.raises(RuntimeError, match="batched handle"):
        capi.Handle.refine(bh, b, x)
    bh.close()
    # Schur handles
    sperm = hostlib.schur_order(prp, pci, np.arange(n - 8, n))
    sprob = LUProblem.from_matrix(prp, pci, np.abs(pv), sperm, relax=8, maxsup=32, nschur=8)
    sh = capi.SchurHandle(sprob, 8)
    with pytest.raises(RuntimeError, match="Schur handle"):
        sh.refine(b, x)
    sh.close()
