"""slu_b200_solve_trans and its doublecomplex / batched twins: A^T x = b and A^H x = b on the factors of A = L U still
resident in HBM, checked against SciPy on F = P A P^T (the ordering of the factored matrix) assembled from the same CSR."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from superlu_dist_b200 import capi
from test_gpu_solve_complex import CASES as ZCASES, complex_csr
from test_gpu_wide_supernodes import _W1
from util import complex_problem, load_fixture, poisson_problem, rel_err

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
RES_TOL = 1e-12     # ||op(F) x - b|| / ||b||
REF_TOL = 1e-10     # against spsolve(op(F), b)

CASES = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=12, leaf=8, relax=16, maxsup=128),
         dict(N=5, leaf=4, relax=8, maxsup=200, fem=3),
         dict(N=16, leaf=16, relax=32, maxsup=256),    # the top separator is one 256-column supernode
         _W1]                                          # 486- and 512-column supernodes (32-vector strips)


def unsym_values(rp, ci, v, seed=0):
    """Non-symmetric values on the pattern: every off-diagonal entry scaled by its own factor in [0.5, 1.5), the diagonal
    set to the row's off-diagonal 1-norm + 1, so the matrix is strictly diagonally dominant (an unpivoted LU exists)."""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    off = rows != ci
    w = np.where(off, np.asarray(v, np.float64) * np.random.default_rng(seed).uniform(0.5, 1.5, len(v)), 0.0)
    return np.where(off, w, np.bincount(rows, np.abs(w), len(rp) - 1)[rows] + 1.0)


def permuted(rp, ci, v, perm):
    """F = P A P^T as a SciPy CSR matrix, perm[old] = new."""
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    perm = np.asarray(perm)
    return sp.csr_matrix((v, (perm[rows], perm[np.asarray(ci)])), shape=(n, n))


def op(F, trans):
    return {"N": F, "T": F.T, "H": F.conj().T}[trans].tocsc()


def check_against_scipy(F, trans, b, x):
    """x solves op(F) x = b: residual and agreement with spsolve, per right-hand side (rows of b)."""
    M = op(F, trans)
    b, x = np.atleast_2d(b), np.atleast_2d(x)
    refs = spl.splu(M).solve(np.ascontiguousarray(b.T)).T
    for bj, xj, ref in zip(b, x, refs):
        res = np.linalg.norm(M @ xj - bj) / np.linalg.norm(bj)
        assert res <= RES_TOL, (trans, res)
        assert rel_err(xj, ref) <= REF_TOL, (trans, rel_err(xj, ref))


def real_case(kw, seed=0):
    """(problem with non-symmetric values in layer 0, rp, ci, values, F)"""
    prob, (rp, ci, v) = poisson_problem(**kw)
    vals = unsym_values(rp, ci, v, seed)
    prob.fill_layer(0, rp, ci, vals)
    return prob, rp, ci, vals, permuted(rp, ci, vals, prob.perm)


@pytest.mark.parametrize("kw", CASES)
def test_transposed_solve_double(kw):
    prob, rp, ci, vals, F = real_case(kw)
    if kw["maxsup"] >= 256:
        assert np.diff(np.asarray(prob.xsup)).max() == kw["maxsup"]
    rng = np.random.default_rng(1)
    b = rng.standard_normal((3, prob.n))
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    for rhs in (b, b[0]):
        x = h.solve(rhs, trans="T")
        assert x.dtype == np.float64 and x.shape == rhs.shape
        check_against_scipy(F, "T", rhs, x)
    xh = h.solve(b[0], trans="H")                    # a real problem: 'H' is 'T'
    check_against_scipy(F, "T", b[0], xh)
    xn = h.solve(b[0])
    check_against_scipy(F, "N", b[0], xn)
    assert rel_err(xn, xh) > 1e-6                    # F is not symmetric: A^T x = b is another system
    h.close()


def test_transposed_solve_unsymmetric_pattern():
    """The reference's unsym360_mmd dump: an unsymmetric pattern whose packed U columns are zero-padded above their
    skyline segments.  Its dense F comes from the panels through prob.matvec of the unit vectors."""
    prob, _, post = load_fixture("unsym360_mmd")
    assert int(post["info"][0]) == 0
    lay = prob.layers[0]
    every = np.ones(prob.nsupers, bool)
    F = prob.matvec([(lay, every)], np.eye(prob.n), 0).T
    assert not np.array_equal(F != 0, (F != 0).T)     # the pattern itself is unsymmetric
    b = np.random.default_rng(2).standard_normal((3, prob.n))
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    for rhs in (b, b[1]):
        x = np.atleast_2d(h.solve(rhs, trans="T"))
        for bj, xj in zip(np.atleast_2d(rhs), x):
            assert np.linalg.norm(F.T @ xj - bj) / np.linalg.norm(bj) <= RES_TOL
            assert rel_err(xj, np.linalg.solve(F.T, bj)) <= REF_TOL
    h.close()


@pytest.mark.parametrize("kw", ZCASES)
def test_transposed_solve_complex(kw):
    """T and H against SciPy; N, T, H, N on one handle: the transposed solves leave the plain one as it was."""
    prob = complex_problem(**kw)
    rp, ci, v = complex_csr(**kw)
    F = permuted(rp, ci, v, prob.perm)
    rng = np.random.default_rng(3)
    b = rng.standard_normal((3, prob.n)) + 1j * rng.standard_normal((3, prob.n))
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    x1 = h.solve(b)
    xs = {}
    for trans in ("T", "H"):
        for rhs in (b, b[0]):
            x = h.solve(rhs, trans=trans)
            assert x.dtype == np.complex128 and x.shape == rhs.shape
            check_against_scipy(F, trans, rhs, x)
        xs[trans] = x
    x2 = h.solve(b)
    check_against_scipy(F, "N", b, x2)
    assert rel_err(xs["T"], xs["H"]) > 1e-6 and rel_err(xs["T"], x2[0]) > 1e-6
    # the plain solve accumulates with atomics, whose order is not fixed: equal up to the last bits
    assert rel_err(x2, x1) <= 1e-14, rel_err(x2, x1)
    h.close()


def test_launches_match_plain_solve():
    for prob in (real_case(CASES[1])[0], complex_problem(**ZCASES[1])):
        h = capi.Handle(prob, 0)
        h.upload()
        assert h.factor() == 0
        b = np.ones(prob.n, prob.dtype)
        counts = {}
        for trans in ("N", "T", "H"):
            h.solve(b, trans=trans)
            st = h.stats()
            assert st.reserved[4] > 0
            counts[trans] = st.reserved[5]
        h.close()
        assert counts["N"] > 0 and counts["T"] == counts["N"] == counts["H"], counts


BKW = [dict(N=12, leaf=8, relax=16, maxsup=128), dict(N=16, leaf=16, relax=32, maxsup=256)]
B = 3


def _batch_members(kw, cplx):
    """(batched problem, rp, ci, (B, nnz) member values, a function j -> an unfactored unbatched problem of member j)"""
    if cplx:
        rp, ci, _ = complex_csr(**kw)
        vals = np.stack([complex_csr(seed=j, **kw)[2] for j in range(B)])
        return complex_problem(**kw), rp, ci, vals, lambda j: complex_problem(seed=j, **kw)
    prob, (rp, ci, v) = poisson_problem(**kw)
    vals = np.stack([unsym_values(rp, ci, v, seed=j) for j in range(B)])
    return prob, rp, ci, vals, lambda j: poisson_problem(**kw)[0]


@pytest.mark.parametrize("kw", BKW)
@pytest.mark.parametrize("cplx", [False, True])
def test_batched_transposed_solve(kw, cplx):
    """Every member's T (and H) solve agrees with an unbatched handle of that member."""
    prob, rp, ci, vals, one = _batch_members(kw, cplx)
    rng = np.random.default_rng(4)
    b = rng.standard_normal((B, 2, prob.n)) + (1j * rng.standard_normal((B, 2, prob.n)) if cplx else 0)
    bh = capi.BatchHandle(prob, B)
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    for trans in ("T", "H") if cplx else ("T",):
        for rhs in (b, b[:, 0]):
            x = bh.solve(rhs, trans=trans)
            assert x.shape == rhs.shape
            for j in range(B):
                p = one(j)
                h = capi.Handle(p, 0)
                h.fill_csr(rp, ci, vals[j], p.perm)
                assert h.factor() == 0
                ref = h.solve(rhs[j], trans=trans)
                h.close()
                assert rel_err(x[j], ref) <= 1e-12, (trans, j, rel_err(x[j], ref))
                check_against_scipy(permuted(rp, ci, vals[j], p.perm), trans, rhs[j], x[j])
    bh.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_batched_transposed_solve_refuses_zero_pivot_member(cplx):
    kw = BKW[0]
    prob, rp, ci, vals, _ = _batch_members(kw, cplx)
    vals[1][np.asarray(prob.perm)[ci] == 0] = 0.0     # column 1 of P A_1 P^T is zero: exact zero pivot there
    bh = capi.BatchHandle(prob, B)
    bh.fill_csr(rp, ci, vals, prob.perm)
    info = bh.factor()
    assert info[1] == 1 and not np.delete(info, 1).any(), info
    for trans in ("T", "H"):
        with pytest.raises(RuntimeError, match="member 1"):
            bh.solve(np.ones((B, prob.n), prob.dtype), trans=trans)
    bh.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_errors(cplx):
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    prob = complex_problem(**kw) if cplx else poisson_problem(**kw)[0]
    L = capi.lib()
    pre = "slu_b200_z_" if cplx else "slu_b200_"
    solve_t, batch_solve_t = getattr(L, pre + "solve_trans"), getattr(L, pre + "batch_solve_trans")
    x = np.ones(prob.n, prob.dtype)
    xp = x.ctypes.data_as(C.c_void_p)
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="needs a successful"):
        h.solve(x, trans="T")                         # not factored yet
    h.upload()
    assert h.factor() == 0
    for t in (3, -1):
        assert solve_t(h.h, xp, prob.n, 1, t) < 0
        assert f"trans = {t}".encode() in L.slu_b200_last_error()
    with pytest.raises(ValueError):
        h.solve(x, trans="C")
    assert batch_solve_t(h.h, xp, prob.n, 1, 1) < 0
    assert b"unbatched handle" in L.slu_b200_last_error()
    h.close()
    bh = capi.BatchHandle(prob, 2)
    with pytest.raises(RuntimeError, match="batch_factor"):
        bh.solve(np.ones((2, prob.n), prob.dtype), trans="T")   # not factored yet
    assert solve_t(bh.h, xp, prob.n, 1, 1) < 0
    assert b"batched handle" in L.slu_b200_last_error()
    rp, ci, v = complex_csr(**kw) if cplx else poisson_problem(**kw)[1]
    bh.fill_csr(rp, ci, np.stack([v, v]), prob.perm)
    assert not bh.factor().any()
    xb = np.ones((2, prob.n), prob.dtype)
    for t in (3, -1):
        assert batch_solve_t(bh.h, xb.ctypes.data_as(C.c_void_p), prob.n, 1, t) < 0
        assert f"trans = {t}".encode() in L.slu_b200_last_error()
    bh.close()


@pytest.mark.parametrize("world", [2, 4])
def test_transposed_solve_1x1xPz(world):
    """The Z-distributed transposed solve, double and doublecomplex, against the single-process result."""
    if capi.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29920 + world), os.path.join(HERE, "mgpu_tsolve_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert out.stdout.count("transposed solve err") == world
