"""slu_b200_z_solve and slu_b200_z_fill_csr: the doublecomplex solve on the factors still resident in HBM (the role of
pzgstrs3d, SRC/complex16/pzgstrs3d.c) and the device-side distribution of a complex CSR matrix."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from superlu_dist_b200 import capi
from util import complex_problem, load_fixture, poisson_problem

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def complex_csr(seed=0, **kw):
    """The matrix of complex_problem(seed, **kw) as CSR in the original ordering: (rowptr, colind, complex128 values),
    built from the same seed the same way.  The permutation to the factored ordering is that problem's .perm."""
    _, (rp, ci, v) = poisson_problem(**kw)
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    vi = np.where(rows == ci, 0.25, 0.5 * rng.uniform(-1.0, 1.0, len(v)))
    return rp, ci, v + 1j * vi

CASES = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=12, leaf=8, relax=16, maxsup=128),
         dict(N=5, leaf=4, relax=8, maxsup=200, fem=3),
         dict(N=16, leaf=16, relax=32, maxsup=256)]   # the top separator is one 256-column supernode


def _crandn(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


@pytest.mark.parametrize("kw", CASES)
def test_complex_solve_on_resident_factors(kw):
    """b = A xtrue in the ordering of the factored matrix; nrhs = 3 and 1; two solves on one handle."""
    prob = complex_problem(**kw)
    A = prob.dense(prob.layers[0], False)
    if kw["maxsup"] == 256:
        assert np.diff(prob.xsup).max() == 256
    rng = np.random.default_rng(3)
    xtrue = _crandn(rng, (3, prob.n))
    b = (A @ xtrue.T).T
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError):
        h.solve(b)                      # not factored yet
    h.upload()
    assert h.factor() == 0
    for rhs, ref in ((b, xtrue), (b[0], xtrue[0])):
        x = h.solve(rhs)
        assert x.dtype == np.complex128 and x.shape == rhs.shape
        err = np.abs(x - ref).max() / np.abs(ref).max()
        assert err <= 1e-10, err
    st = h.stats()
    assert st.reserved[4] > 0 and st.reserved[5] > 0
    h.close()


def test_complex_solve_reference_matrix():
    """The reference's own complex matrix (cg20 through pzdrive3d): factor, solve, residual."""
    prob, _, post = load_fixture("cg20_pzdrive3d")
    assert int(post["info"][0]) == 0
    A = prob.dense(prob.layers[0], False)
    b = _crandn(np.random.default_rng(4), (2, prob.n))
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    x = h.solve(b)
    h.close()
    res = np.linalg.norm(A @ x.T - b.T) / np.linalg.norm(b)
    assert res <= 1e-12, res


@pytest.mark.parametrize("kw", [CASES[0], CASES[2]])
def test_complex_device_side_distribution(kw):
    """slu_b200_z_fill_csr puts into HBM exactly the values the host-distributed layer holds (bit for bit); then
    factor and solve from it."""
    prob = complex_problem(**kw)
    rp, ci, v = complex_csr(**kw)
    want = prob.layers[0].copy()
    A = prob.dense(want, False)
    prob.layers[0].lval[:] = -7.0 - 7.0j              # poison the host arrays: they must not be read
    prob.layers[0].uval[:] = -7.0 - 7.0j
    h = capi.Handle(prob, 0)
    h.fill_csr(rp, ci, v, prob.perm)
    h.download()
    assert np.array_equal(prob.layers[0].lval.view(np.uint64), want.lval.view(np.uint64))
    assert np.array_equal(prob.layers[0].uval.view(np.uint64), want.uval.view(np.uint64))
    assert h.factor() == 0
    xtrue = _crandn(np.random.default_rng(5), (2, prob.n))
    x = h.solve((A @ xtrue.T).T)
    h.close()
    err = np.abs(x - xtrue).max() / np.abs(xtrue).max()
    assert err <= 1e-10, err


def test_complex_solve_argument_errors():
    prob = complex_problem(**CASES[0])
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    n = prob.n
    x = np.zeros((2, n), np.complex128)
    ptr = x.ctypes.data_as(C.c_void_p)
    solve = capi.lib().slu_b200_z_solve
    with pytest.raises(RuntimeError):
        capi._check(solve(h.h, ptr, n, 0))         # nrhs < 1
    with pytest.raises(RuntimeError):
        capi._check(solve(h.h, ptr, n - 1, 1))     # ldx < n
    capi._check(solve(h.h, ptr, n, 2))             # the handle is still usable: zero right-hand sides give zero
    assert not np.any(x)
    h.close()


@pytest.mark.parametrize("world", [2, 4])
def test_complex_solve_1x1xPz(world):
    """The Z-distributed complex solve: every rank passes the same b and receives the full x."""
    if capi.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29900 + world), os.path.join(HERE, "mgpu_zsolve_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert out.stdout.count("complex solve err") == world
