"""Gradients through solves and log-determinants on the resident factors: slu_b200_selinv_device, _logdet_device,
_logdet_grad_device, _solve_grad_device and their batched and doublecomplex twins, and superlu_dist_b200.autograd on top of
them.  gradcheck; the gradients against dense torch.linalg.solve / slogdet; the kernels against NumPy restatements; a GMRF
hyper-parameter step; no host wait; one CUDA graph of a whole step replayed with new values; a zero-pivot member; the
refusals."""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.sparse as sp

from superlu_dist_b200 import LUProblem, autograd, capi, hostlib
from test_gpu_device_io import SLEEP_CYCLES, members, rhs, setup, stream_ptr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
B = 4
U = 2.0 ** -53
NONDET_TOL = 1e-12     # the solves sum with atomics: two backward passes agree to rounding, not bit for bit
CASES = [(name, cplx, batched) for name in ("matgen", "kkt") for cplx in (False, True) for batched in (False, True)]
IDS = [f"{n}-{'z' if c else 'd'}-{'B4' if b else 'B1'}" for n, c, b in CASES]


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


def prepared(name, cplx, batched, seed=3):
    """a handle after the scaled fill of setup()'s matrix (B value sets when batched), and what it was filled with"""
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    V = members(rp, ci, v1, seed) if batched else v1
    h = capi.BatchHandle(prob, B) if batched else capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, V, prob.perm, prs[0], R0, C0)
    return h, prob, rp, ci, V


def dense(rp, ci, v, n):
    """the dense A of each member: (n, n) or (B, n, n) torch CPU tensors"""
    V = np.atleast_2d(v)
    out = np.stack([sp.csr_matrix((V[j], ci, rp), shape=(n, n)).toarray() for j in range(V.shape[0])])
    return torch.from_numpy(out if np.ndim(v) == 2 else out[0])


def scatter_grad(G, rp, ci):
    """a dense gradient sampled on the pattern, in CSR entry order: (..., nnz)"""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    return G[..., rows, ci]


def cond(rp, ci, v, n):
    A = dense(rp, ci, v, n).numpy()
    return float(np.max(np.linalg.cond(A)))


# ---- 1. against dense torch ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
@pytest.mark.parametrize("nrhs", [1, 5])
def test_gradients_match_dense_torch(name, cplx, batched, nrhs):
    h, prob, rp, ci, V = prepared(name, cplx, batched)
    n = prob.n
    lead = (B,) if batched else ()
    shape = lead + ((n,) if nrhs == 1 else (nrhs, n))
    b0, w0 = rhs(shape, cplx, 5), rhs(shape, cplx, 6)
    val = cuda(V).requires_grad_()
    b = cuda(b0).requires_grad_()
    f = autograd.factorize(h, val)
    x = f.solve(b)
    sign, logabs = f.slogdet()
    loss = (cuda(w0) * x).real.sum() + logabs.sum()
    if cplx:
        loss = loss + (cuda(np.full(sign.shape, 0.3 - 0.7j)) * sign).real.sum()
    loss.backward()
    # dense reference on the CPU
    A = dense(rp, ci, V, n).requires_grad_()
    bt = torch.from_numpy(b0).requires_grad_()
    bb = bt if nrhs == 1 else bt.transpose(-1, -2)
    xt = torch.linalg.solve(A, bb.unsqueeze(-1) if nrhs == 1 else bb)
    xt = xt.squeeze(-1) if nrhs == 1 else xt.transpose(-1, -2)
    st, lt = torch.linalg.slogdet(A)
    lref = (torch.from_numpy(w0) * xt).real.sum() + lt.sum()
    if cplx:
        lref = lref + (torch.from_numpy(np.full(st.shape, 0.3 - 0.7j)) * st).real.sum()
    lref.backward()
    gA = scatter_grad(A.grad.numpy(), rp, ci)
    # first-order perturbation: both sides carry errors of order n u cond(A) relative to the gradient's size
    tol = 64 * n * U * cond(rp, ci, V, n)
    assert np.abs(host(val.grad) - gA).max() <= tol * np.abs(gA).max(), (name, np.abs(host(val.grad) - gA).max() / np.abs(gA).max(), tol)
    assert np.abs(host(b.grad) - bt.grad.numpy()).max() <= tol * np.abs(bt.grad.numpy()).max()
    assert np.allclose(host(logabs), lt.detach().numpy(), rtol=1e-12, atol=1e-12)
    assert np.allclose(host(sign), st.detach().numpy(), rtol=1e-12, atol=1e-12)
    h.close()


# ---- 2. gradcheck --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("batched", [False, True])
def test_gradcheck(cplx, batched):
    h, prob, rp, ci, V = prepared("kkt", cplx, batched)
    n = prob.n
    lead = (B,) if batched else ()
    val = cuda(V).requires_grad_()
    handles = [h]

    def fresh():
        # gradcheck differentiates its first evaluation after the perturbed ones: one handle per evaluation keeps each
        # evaluation's factors alive
        handles.append(prepared("kkt", cplx, batched)[0])
        return handles[-1]

    for nrhs in (1, 5):
        b = cuda(rhs(lead + ((n,) if nrhs == 1 else (nrhs, n)), cplx, 8)).requires_grad_()
        assert torch.autograd.gradcheck(lambda v, bb: autograd.factorize(fresh(), v).solve(bb), (val, b), fast_mode=True, eps=1e-6,
                                        atol=1e-6, rtol=1e-5, nondet_tol=NONDET_TOL)
    if cplx:
        fn = lambda v: autograd.factorize(fresh(), v).slogdet()          # noqa: E731  (the phase is differentiable)
    else:
        fn = lambda v: autograd.factorize(fresh(), v).slogdet()[1]       # noqa: E731
    assert torch.autograd.gradcheck(fn, (val,), fast_mode=True, eps=1e-6, atol=1e-6, rtol=1e-5, nondet_tol=NONDET_TOL)
    for x in handles:
        x.close()


# ---- 3. the kernels against NumPy ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
def test_kernels_restated(name, cplx, batched):
    h, prob, rp, ci, V = prepared(name, cplx, batched)
    n, nnz = prob.n, len(ci)
    Bm = B if batched else 1
    info = h.factor()
    assert (np.atleast_1d(info) == 0).all()
    rows = np.repeat(np.arange(n), np.diff(rp))
    # solve_grad: componentwise |g - g_ref| <= 2 nrhs u sum_k |lam_ik| |x_jk|
    for nrhs in (1, 8):
        lead = (B,) if batched else ()
        lam, x = rhs(lead + (nrhs, n), cplx, 11), rhs(lead + (nrhs, n), cplx, 12)
        if nrhs == 1:
            lam, x = lam[..., 0, :], x[..., 0, :]
        g = host(h.solve_grad(cuda(lam), cuda(x))).reshape(Bm, nnz)
        L3, X3 = lam.reshape(Bm, nrhs, n), x.reshape(Bm, nrhs, n)
        ref = -np.einsum("mki,mki->mi", L3[:, :, rows], np.conj(X3[:, :, ci]))
        bound = 2 * nrhs * U * np.einsum("mki,mki->mi", np.abs(L3[:, :, rows]), np.abs(X3[:, :, ci]))
        assert (np.abs(g - ref) <= bound * (2 if cplx else 1)).all(), (name, nrhs)
    # selinv_device and logdet_device: bit for bit the host calls
    if batched:
        perm_r = h_perm_r = None
        RC = [h.scaling(j) for j in range(B)]
    else:
        h_perm_r, R, Cs = h.scaling()
        RC = [(R, Cs)]
    perm_r = h_perm_r if h_perm_r is not None else setup(name, cplx)[5][0]
    pF, qF = prob.perm[perm_r[rows]], prob.perm[ci]     # entry e = (i, j) sits at F(pF, qF)
    order = np.lexsort((pF, qF))
    srp = np.concatenate([[0], np.cumsum(np.bincount(qF, minlength=n))]).astype(np.int32)
    ident = np.arange(n, dtype=np.int32)
    h.selinv()
    Hs = np.empty((Bm, nnz), np.complex128 if cplx else np.float64)
    Hs[:, order] = np.asarray(h.inv_entries(srp, pF[order].astype(np.int32), ident)).reshape(Bm, nnz)   # H(pF, qF)
    sg_h, la_h = h.logdet()
    torch.cuda.synchronize()
    h.selinv_device()
    sg_d, la_d = h.logdet_device()
    torch.cuda.synchronize()
    Hd = np.empty_like(Hs)
    Hd[:, order] = np.asarray(h.inv_entries(srp, pF[order].astype(np.int32), ident)).reshape(Bm, nnz)
    assert np.array_equal(Hd, Hs), name
    assert np.array_equal(np.atleast_1d(host(la_d)), np.atleast_1d(la_h)) and np.array_equal(np.atleast_1d(host(sg_d)), np.atleast_1d(sg_h))
    # logdet_grad: c ((R_i conj(h)) C_j), every multiply and add rounded on its own
    coef = rhs((Bm,), cplx, 13)
    g = host(h.logdet_grad(cuda(coef if batched else coef[:1]))).reshape(Bm, nnz)
    for j in range(Bm):
        R, Cs = RC[j]
        hh = np.conj(Hs[j]) if cplx else Hs[j]
        if cplx:
            ux, uy = (R[rows] * hh.real) * Cs[ci], (R[rows] * hh.imag) * Cs[ci]
            ref = (coef[j].real * ux - coef[j].imag * uy) + 1j * (coef[j].real * uy + coef[j].imag * ux)
        else:
            ref = coef[j] * ((R[rows] * hh) * Cs[ci])
        assert np.array_equal(g[j], ref), (name, j)
    assert h.stats().reserved[5] == 1
    h.close()


# ---- 4. a GMRF hyper-parameter step --------------------------------------------------------------------------------------
def test_gmrf_hyperparameter_gradient():
    rp, ci, kv = hostlib.poisson3d(6)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    iv = (rows == ci).astype(np.float64)
    perm = hostlib.nd_order(6, leaf=8)
    prob = LUProblem.from_matrix(rp, ci, kv, perm, relax=8, maxsup=32)
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, kv + iv, perm, equil=False)
    b0 = rhs(n, False, 21)
    theta = torch.tensor([0.7, 1.3], dtype=torch.float64, device="cuda", requires_grad=True)
    K, I, b = cuda(kv), cuda(iv), cuda(b0)
    f = autograd.factorize(h, theta[0] * K + theta[1] * I)
    L = 0.5 * f.slogdet()[1] - 0.5 * (b * f.solve(b)).sum()
    L.backward()
    th = torch.tensor([0.7, 1.3], dtype=torch.float64, requires_grad=True)
    Q = th[0] * dense(rp, ci, kv, n) + th[1] * torch.eye(n, dtype=torch.float64)
    bt = torch.from_numpy(b0)
    Lt = 0.5 * torch.linalg.slogdet(Q)[1] - 0.5 * (bt * torch.linalg.solve(Q, bt)).sum()
    Lt.backward()
    assert np.allclose(host(theta.grad), th.grad.numpy(), rtol=1e-10, atol=0), (host(theta.grad), th.grad.numpy())
    h.close()


# ---- 5. no host wait -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
def test_no_host_wait(cplx):
    h, prob, rp, ci, V = prepared("kkt", cplx, False)
    n = prob.n
    val = cuda(V)
    lam, x = cuda(rhs((3, n), cplx, 1)), cuda(rhs((3, n), cplx, 2))
    coef = cuda(rhs((1,), cplx, 3))

    def calls():
        h.refill(val)
        h.factor_device()
        h.selinv_device()
        out = h.logdet_device()
        return out, h.logdet_grad(coef), h.solve_grad(lam, x)

    calls()                                  # the first calls allocate
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    t0 = time.perf_counter()
    out = calls()
    dt = time.perf_counter() - t0
    pending = not torch.cuda.current_stream().query()
    torch.cuda.synchronize()
    assert pending and dt < 0.02, dt
    sg, la = h.logdet()                      # a host call after the device sweep: the inverse is usable
    assert float(host(out[0][1])) == la
    h.inv_diag()
    h.close()


# ---- 6. one CUDA graph of a whole step -----------------------------------------------------------------------------------
def step(h, sv, sb, w):
    f = autograd.factorize(h, sv)
    x = f.solve(sb)
    _, logabs = f.slogdet()
    loss = (w * x).real.sum() + logabs.sum()
    return torch.autograd.grad(loss, (sv, sb))


@pytest.mark.parametrize("cplx,batched", [(False, False), (True, False), (False, True), (True, True)], ids=["d-B1", "z-B1", "d-B4", "z-B4"])
def test_graph_replay(cplx, batched):
    h, prob, rp, ci, V = prepared("matgen", cplx, batched)
    e, *_ = prepared("matgen", cplx, batched)
    n = prob.n
    lead = (B,) if batched else ()
    sv = cuda(V).requires_grad_()
    sb = cuda(rhs(lead + (2, n), cplx, 1)).requires_grad_()
    w = cuda(rhs(lead + (2, n), cplx, 2))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(h, sv, sb, w)                   # warm-up outside capture: slot map, inverse arena, buffers
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step(h, sv, sb, w)
    for it, seed in enumerate((31, 32)):
        Vn = members(rp, ci, setup("matgen", cplx)[4], seed) if batched else setup("matgen", cplx)[4] * (1 + 0.1 * it)
        bn = rhs(lead + (2, n), cplx, seed)
        with torch.no_grad():
            sv.copy_(cuda(Vn))
            sb.copy_(cuda(bn))
        g.replay()
        torch.cuda.synchronize()
        ref = step(e, cuda(Vn).requires_grad_(), cuda(bn).requires_grad_(), w)
        for a, r in zip(out, ref):
            assert np.abs(host(a) - host(r)).max() <= 1e-10 * np.abs(host(r)).max(), it
    del g
    h.close()
    e.close()
    # a first selinv_device under capture is refused, and the capture stays valid
    h, *_ = prepared("kkt", cplx, batched)
    h.factor()
    y = cuda(np.arange(4.0))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        with pytest.raises(RuntimeError, match="first selected inversion"):
            h.selinv_device()
        z = y * 2
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(host(z), 2 * np.arange(4.0))
    h.close()


# ---- 7. a member with an exact zero pivot; refusals ----------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
def test_zero_pivot_member(cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("matgen", cplx)
    n = prob.n
    W = members(rp, ci, v1, 3)
    row = n // 3
    bad = 1
    Z = W.copy()
    Z[bad, rp[row]:rp[row + 1]] = 0
    grads = []
    for vals in (Z, W):
        h = capi.BatchHandle(prob, B)
        h.fill_csr_scaled(rp, ci, W, prob.perm, prs[0], R0, C0)
        val = cuda(vals).requires_grad_()
        f = autograd.factorize(h, val)
        loss = f.solve(cuda(rhs((B, n), cplx, 4))).real.sum() + f.slogdet()[1].sum()
        loss.backward()
        grads.append(host(val.grad))
        h.close()
    assert np.isnan(grads[0][bad]).all()
    for j in range(B):
        if j != bad:
            assert np.abs(grads[0][j] - grads[1][j]).max() <= 1e-12 * np.abs(grads[1][j]).max(), j


@pytest.mark.parametrize("cplx", [False, True])
def test_refusals(cplx):
    h, prob, rp, ci, V = prepared("kkt", cplx, False)
    n = prob.n
    val = cuda(V).requires_grad_()
    f = autograd.factorize(h, val)
    x = f.solve(cuda(rhs(n, cplx, 1)))
    la = f.slogdet()[1]
    h.refill(cuda(V))                          # the factors of f are gone
    with pytest.raises(RuntimeError, match="replaced by Handle.refill"):
        x.real.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="replaced by Handle.refill"):
        la.backward()
    f = autograd.factorize(h, val)
    x = f.solve(cuda(rhs(n, cplx, 1)))
    h.factor()
    with pytest.raises(RuntimeError, match="replaced by Handle.factor"):
        x.real.sum().backward()
    # the host knows the inverse is stale
    h.factor()
    with pytest.raises(RuntimeError, match="selinv_device or"):
        h.logdet_grad(cuda(rhs((1,), cplx, 2)))
    # host pointers through the raw call
    fn = capi._fn("logdet_grad_device", cplx)
    h.selinv_device()
    g = torch.zeros(len(ci), dtype=val.dtype, device="cuda")
    hc = np.ones(2)
    assert fn(h.h, capi._ptr(hc), C.c_void_p(g.data_ptr()), stream_ptr()) != 0
    assert "coef must point at device or managed memory" in capi.lib().slu_b200_last_error().decode()
    h.close()
    # an unscaled handle
    prob2, rp2, ci2, v1, _, prs, _, _ = setup("kkt", cplx)
    hp = capi.Handle(prob2, 0)
    hp.fill_csr(*hostlib.row_permute(rp2, ci2, v1, prs[0]), prob2.perm)
    assert hp.factor() == 0
    with pytest.raises(RuntimeError, match="scaled fill"):
        hp.selinv_device()
    with pytest.raises(RuntimeError, match="scaled fill"):
        hp.logdet_device()
    hp.close()
    # a Schur handle
    prp, pci, pv = hostlib.row_permute(rp2, ci2, v1, prs[0])
    sperm = hostlib.schur_order(prp, pci, np.arange(n - 8, n))
    sprob = LUProblem.from_matrix(prp, pci, np.abs(pv), sperm, relax=8, maxsup=32, nschur=8)
    if cplx:
        sprob.dtype = np.dtype(np.complex128)
        for lay in sprob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    sh = capi.SchurHandle(sprob, 8)
    with pytest.raises(RuntimeError, match="Schur handle"):
        sh.selinv_device()
    sh.close()
