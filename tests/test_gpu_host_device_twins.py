"""The host-synchronous gsrfs / gscon after a captured call of the other kind on the caller's stream.  A captured
gsrfs_device without ferr leaves the estimator's buffers unallocated, and a captured gscon_device leaves the refinement's:
no graph holds them, so the first host call that needs them allocates them instead of being refused as if it would move a
buffer a graph uses.  Double and doublecomplex, unbatched and B = 4."""
import numpy as np
import pytest

from test_gpu_device_io import rhs
from test_gpu_refine_device import RCOND_TOL, check_refinement, cuda, handle, prepared

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
B = 4
CASES = [(cplx, batched) for cplx in (False, True) for batched in (False, True)]
IDS = [f"{'z' if c else 'd'}-{'B4' if b else 'B1'}" for c, b in CASES]


@pytest.mark.parametrize("cplx,batched", CASES, ids=IDS)
def test_host_gscon_after_captured_gsrfs_device(cplx, batched):
    h, prob, rp, ci, V, prs, R0, C0 = prepared("kkt", cplx, batched)
    b = rhs((B, 2, prob.n) if batched else (2, prob.n), cplx, 5)
    bd, xd = cuda(b), cuda(h.solve_scaled(b))
    h.refine(bd, xd, ferr=False)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        h.refine(bd, xd, ferr=False)
    torch.cuda.synchronize()
    anorm = np.array([1.7, 2.0, 2.5, 3.2]) if batched else 1.7
    rc = h.rcond(anorm)
    e = handle(prob, batched)                       # the same factors on a handle without a capture
    e.fill_csr_scaled(rp, ci, V, prob.perm, prs[0], R0, C0)
    assert (np.atleast_1d(e.factor()) == 0).all()
    ref = e.rcond(anorm)
    assert np.allclose(rc, ref, rtol=RCOND_TOL, atol=0), (rc, ref)
    del g
    h.close()
    e.close()


@pytest.mark.parametrize("cplx,batched", CASES, ids=IDS)
def test_host_refine_after_captured_gscon_device(cplx, batched):
    h, prob, rp, ci, V, *_ = prepared("kkt", cplx, batched)
    b = rhs((B, prob.n) if batched else prob.n, cplx, 5)
    x0 = h.solve_scaled(b)
    an = cuda(np.full(B if batched else 1, 2.5))
    h.rcond(an)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        h.rcond(an)
    torch.cuda.synchronize()
    x, berr, steps, ferr = h.refine(b, x0)
    col = (lambda a: a[:, None]) if batched else (lambda a: np.atleast_1d(a)[None])
    check_refinement(rp, ci, V, col(b), col(x), col(berr), col(steps), col(ferr), batched)
    del g
    h.close()
