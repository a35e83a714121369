"""Kernel-level parity through the C-ABI (include/slu_b200.h, slu_b200_k_*): each hand-written
sm_90a kernel against a NumPy/SciPy restatement of the same BLAS-level operation the reference
calls (dger-based LU pdgstrf2.c:508-601, dtrsm dtrfCommWrapper.c:166-219 / pdgstrf2.c:832, dgemm
dscatter3d.c:143).  FP64 tolerance 1e-12 relative to the result's magnitude times the size."""
import numpy as np
import pytest
import scipy.linalg as sl

from superlu_dist_b200 import capi

pytestmark = pytest.mark.gpu


def lu_nopivot(a):
    a = a.copy()
    n = a.shape[1]
    for j in range(n - 1):
        if a[j, j] != 0:
            a[j + 1:n, j] /= a[j, j]
        a[j + 1:n, j + 1:] -= np.outer(a[j + 1:n, j], a[j, j + 1:])
    return a


@pytest.mark.parametrize("ns,extra", [(1, 0), (5, 3), (16, 0), (17, 40), (33, 7), (48, 0), (65, 2), (96, 0), (100, 1),
                                      (129, 30), (200, 0), (240, 5), (255, 1), (256, 19), (300, 0)])
def test_diag_lu(ns, extra):
    """Blocks of 65..256 columns take the 8-CTA cluster kernel, the others the one-CTA kernel."""
    rng = np.random.default_rng(ns)
    a = rng.standard_normal((ns + extra, ns))
    a[:ns] += ns * np.eye(ns)
    ref = a.copy()
    ref[:ns] = lu_nopivot(a[:ns])
    out, info, tiny = capi.k_diag_lu(a)
    assert info == 0 and tiny == 0
    assert np.abs(out - ref).max() <= 1e-12 * ns * np.abs(ref).max()


def test_diag_lu_tiny_and_zero_pivot():
    rng = np.random.default_rng(3)
    a = rng.standard_normal((40, 40)) + 40 * np.eye(40)
    a[0, 0] = 1e-30
    out, info, tiny = capi.k_diag_lu(a.copy(), replace_tiny=1, thresh=1e-3)
    b = a.copy()
    b[0, 0] = 1e-3
    assert tiny >= 1 and info == 0
    assert np.abs(out - lu_nopivot(b)).max() <= 1e-9 * np.abs(lu_nopivot(b)).max()
    a = rng.standard_normal((8, 8)) + 8 * np.eye(8)
    a[:, 0] = 0.0   # exact zero pivot at column 0 (and it stays zero)
    out, info, tiny = capi.k_diag_lu(a.copy(), col0=100)
    assert info == 101  # 1-based global column, pdgstrf2.c:568-571
    # the same inside a block wide enough for the cluster kernel (ns >= 65), past its first 32-column slab
    a = rng.standard_normal((100, 100)) + 100 * np.eye(100)
    a[70, 70] = 1e-30
    a[:70, 70] = 0.0
    a[70, :70] = 0.0
    out, info, tiny = capi.k_diag_lu(a.copy(), replace_tiny=1, thresh=1e-3)
    b = a.copy()
    b[70, 70] = 1e-3
    assert tiny >= 1 and info == 0
    assert np.abs(out - lu_nopivot(b)).max() <= 1e-9 * np.abs(lu_nopivot(b)).max()
    a = rng.standard_normal((90, 90)) + 90 * np.eye(90)
    a[:, 40] = 0.0
    a[40, :] = 0.0
    out, info, tiny = capi.k_diag_lu(a.copy(), col0=1000)
    assert info == 1041


@pytest.mark.parametrize("ns,m", [(1, 1), (7, 3), (16, 64), (31, 65), (64, 200), (256, 130), (300, 70)])
def test_trsm_l(ns, m):
    rng = np.random.default_rng(ns * 1000 + m)
    lu = rng.standard_normal((ns, ns)) + ns * np.eye(ns)
    x = rng.standard_normal((m, ns))
    ref = sl.solve_triangular(np.triu(lu), x.T, trans="T", lower=False).T   # X U^-1
    out = capi.k_trsm(lu, x, ucase=False)
    assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1)


@pytest.mark.parametrize("ns,nc", [(1, 1), (7, 3), (16, 64), (31, 65), (64, 200), (256, 130), (300, 70)])
def test_trsm_u(ns, nc):
    rng = np.random.default_rng(ns * 1000 + nc + 7)
    lu = rng.standard_normal((ns, ns)) / ns + np.eye(ns)
    x = rng.standard_normal((ns, nc))
    ref = sl.solve_triangular(np.tril(lu, -1) + np.eye(ns), x, lower=True, unit_diagonal=True)
    out = capi.k_trsm(lu, x, ucase=True)
    assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1)


@pytest.mark.parametrize("m,n,k", [(1, 1, 1), (7, 5, 3), (33, 31, 17), (96, 96, 16), (128, 128, 4), (130, 257, 100),
                                   (300, 200, 256), (95, 400, 30), (513, 129, 33)])
def test_gemm_sub(m, n, k):
    rng = np.random.default_rng(m * 7 + n * 3 + k)
    a, b, c = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((m, n))
    out, _ = capi.k_gemm_sub(a, b, c)
    ref = c - a @ b
    assert np.abs(out - ref).max() <= 1e-13 * k * max(np.abs(ref).max(), 1)
