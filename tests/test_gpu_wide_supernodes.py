"""Supernodes up to MAX_SUPER_SIZE = 512 columns (SRC/include/superlu_defs.h:154; sp_ienv(3) may be raised to it by the
caller through SUPERLU_MAXSUP): panel solves with 32-vector strips above 416 columns, the one-CTA diagonal LU, the FP64
DMMA and the int8 tensor-core Schur paths with k up to 512, and the resident solve -- kernel level against SciPy, whole
factorization against the oracle (same tolerances as test_gpu_kernels.py / test_gpu_parity.py)."""
import numpy as np
import pytest
import scipy.linalg as sl

from oracle import oracle
from superlu_dist_b200 import capi
from util import poisson_problem, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10


def _lu_nopivot(a):
    a = a.copy()
    n = a.shape[1]
    for j in range(n - 1):
        a[j + 1:n, j] /= a[j, j]
        a[j + 1:n, j + 1:] -= np.outer(a[j + 1:n, j], a[j, j + 1:])
    return a


@pytest.mark.parametrize("ns,extra", [(417, 5), (486, 0), (512, 33)])
def test_diag_lu_wide(ns, extra):
    rng = np.random.default_rng(ns)
    a = rng.standard_normal((ns + extra, ns))
    a[:ns] += ns * np.eye(ns)
    ref = a.copy()
    ref[:ns] = _lu_nopivot(a[:ns])
    out, info, tiny = capi.k_diag_lu(a)
    assert info == 0 and tiny == 0
    assert np.abs(out - ref).max() <= 1e-12 * ns * np.abs(ref).max()


@pytest.mark.parametrize("ns,m", [(416, 70), (417, 1), (432, 33), (486, 100), (512, 64), (512, 257)])
def test_trsm_wide(ns, m):
    """416 is the last width on 64-vector strips; everything above takes 32-vector strips."""
    rng = np.random.default_rng(ns * 1000 + m)
    lu = rng.standard_normal((ns, ns)) + ns * np.eye(ns)
    x = rng.standard_normal((m, ns))
    ref = sl.solve_triangular(np.triu(lu), x.T, trans="T", lower=False).T   # X U^-1
    out = capi.k_trsm(lu, x, ucase=False)
    assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1)
    lu = rng.standard_normal((ns, ns)) / ns + np.eye(ns)
    x = rng.standard_normal((ns, m))
    ref = sl.solve_triangular(np.tril(lu, -1) + np.eye(ns), x, lower=True, unit_diagonal=True)
    out = capi.k_trsm(lu, x, ucase=True)
    assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1)


_W1 = dict(N=18, leaf=32, relax=64, maxsup=512, fem=3)   # supernodes of 486, 512, 512 columns, two of them below the root
_W2 = dict(N=24, leaf=32, relax=64, maxsup=512)          # 576-column top separator -> 512 + 64


@pytest.mark.parametrize("kw,tc_slices", [(_W1, -1), (_W1, 7), (_W2, -1), (_W2, 7)])
def test_factorization_with_wide_supernodes(kw, tc_slices):
    """tc_slices = -1: FP64 DMMA Schur only; 7: the int8 tensor-core path (16 k-steps at 512 columns)."""
    prob, _ = poisson_problem(**kw)
    chk, _ = poisson_problem(**kw)
    assert np.diff(np.asarray(prob.xsup)).max() == 512
    info, st = capi.pdgstrf3d(prob, 0, tc_slices=tc_slices, tc_min_ns=64)
    oinfo, oops, _ = oracle.factor(chk)
    assert info == oinfo == 0
    assert (st.reserved[1] > 0) == (tc_slices > 0)
    assert abs(st.ops_fact - oops) <= 1e-9 * oops
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL


def test_solve_with_wide_supernodes():
    prob, _ = poisson_problem(**_W1)
    lay = prob.layers[0]
    every = np.ones(prob.nsupers, bool)
    xtrue = np.random.default_rng(2).standard_normal((2, prob.n))
    b = prob.matvec([(lay, every)], xtrue, 0)
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    x = h.solve(b)
    assert np.abs(x - xtrue).max() <= 1e-10 * np.abs(xtrue).max()
    h.close()
