"""Panel TRSM (trsm_kernel, slu_b200_k_trsm_l / _u) at the edges of its tiling: one 32-vector strip per CTA, 16-column
blocks on DMMA.16x8x8 and T streamed in 64-row chunks.  Widths that are not a multiple of 16 (1, 15, 17, 255, 257,
417) leave a partial last block, 255..512 span several T chunks per block, and vector counts that are not a multiple of
the strip leave a partial last strip.  Against SciPy, with the tolerance of test_gpu_kernels.py."""
import numpy as np
import pytest
import scipy.linalg as sl

from superlu_dist_b200 import capi

pytestmark = pytest.mark.gpu

CASES = [(1, 1), (15, 33), (17, 95), (255, 64), (256, 32), (256, 1000), (257, 95), (416, 31), (417, 65), (512, 97)]


@pytest.mark.parametrize("ns,m", CASES)
def test_trsm_l_strips(ns, m):
    rng = np.random.default_rng(ns * 1000 + m + 3)
    lu = rng.standard_normal((ns, ns)) + ns * np.eye(ns)
    x = rng.standard_normal((m, ns))
    ref = sl.solve_triangular(np.triu(lu), x.T, trans="T", lower=False).T   # X U^-1
    out = capi.k_trsm(lu, x, ucase=False)
    assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1)


@pytest.mark.parametrize("ns,nc", CASES)
def test_trsm_u_strips(ns, nc):
    rng = np.random.default_rng(ns * 1000 + nc + 11)
    lu = rng.standard_normal((ns, ns)) / ns + np.eye(ns)
    x = rng.standard_normal((ns, nc))
    ref = sl.solve_triangular(np.tril(lu, -1) + np.eye(ns), x, lower=True, unit_diagonal=True)
    out = capi.k_trsm(lu, x, ucase=True)
    assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1)
