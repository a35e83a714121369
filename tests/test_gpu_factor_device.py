"""Factorization on the caller's CUDA stream and CUDA graphs of refill -> factor -> solve: slu_b200_factor_device, its
batched and doublecomplex twins, through Handle / BatchHandle.factor_device and the raw C calls.  The device factors against
the host factorization's; the device status, the NaN guard of the device solves and the host refusals after a zero pivot;
no host wait and the stream order; torch.cuda.CUDAGraph replays against eager iterations; the capture refusals and the
pinned buffers; the argument refusals."""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.sparse as sp

from superlu_dist_b200 import LUProblem, capi, hostlib
from test_gpu_device_io import AGREE_TOL, B, RES_TOL, SLEEP_CYCLES, cuda, members, rel, rhs, setup, stream_ptr
from test_gpu_static_pivot import arena, residual

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
CASES = [(name, cplx, batched) for name in ("matgen", "kkt") for cplx in (False, True) for batched in (False, True)]
IDS = [f"{n}-{'z' if c else 'd'}-{'B4' if b else 'B1'}" for n, c, b in CASES]


def handle(prob, batched, **opt):
    return capi.BatchHandle(prob, B, **opt) if batched else capi.Handle(prob, 0, **opt)


def values(rp, ci, v, batched, seed):
    return members(rp, ci, v, seed) if batched else v


def arenas(h, prob, batched):
    out = []
    for j in range(B if batched else 1):
        h.download(j) if batched else h.download()
        out.append(arena(prob))
    return out


def error_of(call):
    with pytest.raises(RuntimeError) as e:
        call()
    return str(e.value)


def matrix(rp, ci, v, n):
    return sp.csr_matrix((v, ci, rp), shape=(n, n))


# ---- 1. the same factors, the same status --------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
def test_device_factors_are_the_host_factors(name, cplx, batched):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    # the equilibrated rows have entries of at most 1: a threshold of 2 replaces at least the first pivot
    prob.replace_tiny_pivot, prob.thresh = 1, 2.0
    V = values(rp, ci, v1, batched, 3)
    hh, hd = handle(prob, batched), handle(prob, batched)
    for h in (hh, hd):
        h.fill_csr_scaled(rp, ci, V, prob.perm, prs[0], R0, C0)
    info_h = np.atleast_1d(hh.factor())
    info_d = hd.factor_device()
    assert info_d.is_cuda and info_d.dtype == torch.int32 and tuple(info_d.shape) == ((B,) if batched else (1,))
    assert (info_d.cpu().numpy() == 0).all() and (info_h == 0).all()
    for a, b in zip(arenas(hh, prob, batched), arenas(hd, prob, batched)):
        assert rel(a[0], b[0]) <= AGREE_TOL and rel(a[1], b[1]) <= AGREE_TOL, name
    sh, sd = hh.stats(), hd.stats()
    assert sh.tiny_pivots > 0 and sd.tiny_pivots == sh.tiny_pivots
    assert sd.t_factor_s == 0 and sd.gpu_launches == sh.gpu_launches + 2
    hh.close()
    hd.close()


# ---- 2. a member with an exact zero pivot --------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
def test_zero_pivot_member(name, cplx, batched):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    n, perm, perm_r = prob.n, prob.perm, prs[0]
    bad = 1 if batched else 0
    V1, V2 = values(rp, ci, v1, batched, 3), np.array(values(rp, ci, v2, batched, 4))
    row = n // 3                                      # a zero row of A: an exact zero pivot in F, whatever the order
    W = np.atleast_2d(V2)
    W[bad, rp[row]:rp[row + 1]] = 0
    V2 = W if batched else W[0]
    hh, hd = handle(prob, batched), handle(prob, batched)
    for h in (hh, hd):
        h.fill_csr_scaled(rp, ci, V1, perm, perm_r, R0, C0)
        h.refill(cuda(V2))
    info_h = np.atleast_1d(hh.factor())
    info_d = hd.factor_device().cpu().numpy()
    assert info_h[bad] > 0 and np.array_equal(info_d, info_h), (info_d, info_h)
    nrhs = 2
    b = rhs((B, nrhs, n) if batched else (nrhs, n), cplx, 7)
    xs = hd.solve_scaled(cuda(b)).cpu().numpy().reshape((-1, nrhs, n))
    xf = hd.solve(cuda(b)).cpu().numpy().reshape((-1, nrhs, n))
    bb = b.reshape((-1, nrhs, n))
    rows = np.repeat(np.arange(n), np.diff(rp))
    for j in range(B if batched else 1):
        if j == bad:
            assert np.isnan(xs[j].real).all() and np.isnan(xf[j].real).all(), j
            if cplx:
                assert np.isnan(xs[j].imag).all() and np.isnan(xf[j].imag).all()
            continue
        vj = np.atleast_2d(V2)[j]
        Rj, Cj = hd.scaling(j) if batched else hd.scaling()[1:]
        F = sp.csr_matrix(((Rj[rows] * vj) * Cj[ci], (perm[perm_r[rows]], perm[ci])), shape=(n, n))
        assert residual(matrix(rp, ci, vj, n), xs[j], bb[j]) <= RES_TOL, (name, j)
        assert residual(F, xf[j], bb[j]) <= RES_TOL, (name, j)
    # the host calls refuse exactly as after the host factorization
    for call in (lambda h: h.rcond(1.0), lambda h: h.solve(b), lambda h: h.solve_scaled(b), lambda h: h.logdet()):
        assert error_of(lambda: call(hd)) == error_of(lambda: call(hh))
    hh.close()
    hd.close()


# ---- 3. no host wait, stream order ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
def test_stream_order_and_no_host_wait(cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("kkt", cplx)
    n = prob.n
    A2 = matrix(rp, ci, v2, n)
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v1, prob.perm, prs[0], R0, C0)
    h.factor_device()
    info = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    t0 = time.perf_counter()
    h.factor_device(info)
    dt = time.perf_counter() - t0
    pending = not torch.cuda.current_stream().query()
    torch.cuda.synchronize()
    assert pending and dt < 0.01, dt
    assert int(info.item()) == 0
    # refill -> factor_device -> solve on a side stream, the values and b written there after a sleep
    side = torch.cuda.Stream()
    src_v, b = cuda(v2), rhs((3, n), cplx, 2)
    src_b = cuda(b)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        vt, bt = torch.zeros_like(src_v), torch.zeros_like(src_b)
        torch.cuda._sleep(SLEEP_CYCLES)
        vt.copy_(src_v)
        bt.copy_(src_b)
        h.refill(vt)
        vt.fill_(float("nan"))                     # after the refill in stream order: the factors are of v2
        inf = h.factor_device()
        y = h.solve_scaled(bt) * 1
    side.synchronize()
    assert int(inf.item()) == 0
    assert residual(A2, y.cpu().numpy(), b) <= RES_TOL
    h.close()


# ---- 4. graph replay -----------------------------------------------------------------------------------------------------
def capture_iteration(h, sv, sb, info):
    """warm-up on a side stream, then one torch.cuda.CUDAGraph of refill -> factor_device -> solve_scaled_device"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        h.refill(sv)
        h.factor_device(info)
        h.solve_scaled(sb)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        h.refill(sv)
        h.factor_device(info)
        sx = h.solve_scaled(sb)
    return g, sx


@pytest.mark.parametrize("lookahead", [True, False], ids=["lookahead", "no_lookahead"])
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
def test_graph_replay(name, cplx, batched, lookahead):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    n = prob.n
    opt = {} if lookahead else {"no_lookahead": 1}
    h, e = handle(prob, batched, **opt), handle(prob, batched, **opt)
    V1 = values(rp, ci, v1, batched, 3)
    for x in (h, e):
        x.fill_csr_scaled(rp, ci, V1, prob.perm, prs[0], R0, C0)
    shape = (B, n) if batched else (n,)
    sv, sb = cuda(values(rp, ci, v2, batched, 4)), cuda(rhs(shape, cplx, 1))
    info = torch.full(((B,) if batched else (1,)), 9, dtype=torch.int32, device="cuda")
    g, sx = capture_iteration(h, sv, sb, info)
    for it in range(3):
        V = np.asarray(values(rp, ci, v2, batched, 20 + it)) * (1.0 + 0.05 * it)
        b = rhs(shape, cplx, 30 + it)
        sv.copy_(cuda(V))
        sb.copy_(cuda(b))
        info.fill_(9)
        g.replay()
        torch.cuda.synchronize()
        x = sx.cpu().numpy()
        assert (info.cpu().numpy() == 0).all()
        e.refill(cuda(V))
        assert (np.atleast_1d(e.factor()) == 0).all()
        xe = e.solve_scaled(b)
        assert rel(x, xe) <= AGREE_TOL, (name, it)
        for j in range(B if batched else 1):
            Vj, xj, bj = (V[j], x[j], b[j]) if batched else (V, x, b)
            assert residual(matrix(rp, ci, Vj, n), xj, bj) <= RES_TOL, (name, it, j)
    sg, la = h.logdet()
    sge, lae = e.logdet()
    assert np.allclose(la, lae, rtol=1e-12, atol=0) and np.allclose(sg, sge, rtol=1e-12, atol=0)
    assert np.allclose(h.rcond(1.0), e.rcond(1.0), rtol=1e-10, atol=0)
    del g
    h.close()
    e.close()


# ---- 5. capture refusals and pinned buffers ------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx,batched", [(False, False), (True, True)], ids=["d-B1", "z-B4"])
def test_capture_refusals_and_pinning(cplx, batched):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("kkt", cplx)
    n = prob.n
    h = handle(prob, batched)
    V1 = values(rp, ci, v1, batched, 3)
    h.fill_csr_scaled(rp, ci, V1, prob.perm, prs[0], R0, C0)
    shape = (B, n) if batched else (n,)
    sv, sb = cuda(values(rp, ci, v2, batched, 4)), cuda(rhs(shape, cplx, 1))
    info = torch.zeros((B,) if batched else (1,), dtype=torch.int32, device="cuda")
    # the first refill after a scaled fill builds the slot map and waits for it: refused under capture, nothing enqueued
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="first refill after a scaled fill builds the slot map"):
        with torch.cuda.graph(g):
            h.refill(sv)
    del g
    # a solve with more right-hand sides than any before would grow d_x
    h.refill(sv)
    h.factor_device(info)
    h.solve_scaled(sb)
    wide = cuda(rhs((B, 3, n) if batched else (3, n), cplx, 2))
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="would allocate device buffers while the stream is capturing"):
        with torch.cuda.graph(g):
            h.solve_scaled(wide)
    del g
    # a good capture pins the buffers
    g, sx = capture_iteration(h, sv, sb, info)
    with pytest.raises(RuntimeError, match="captured CUDA graph"):
        h.solve_scaled(rhs((B, 3, n) if batched else (3, n), cplx, 3))
    keep = np.ones(len(ci), bool)
    rows = np.repeat(np.arange(n), np.diff(rp))
    keep[np.flatnonzero(rows != ci)[0]] = False                  # one off-diagonal entry less: another nnz
    rp2 = np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=n))]).astype(np.int32)
    V1k = np.atleast_2d(V1)[:, keep]
    with pytest.raises(RuntimeError, match="captured CUDA graph"):
        h.fill_csr_scaled(rp2, ci[keep], V1k if batched else V1k[0], prob.perm, prs[0], R0, C0)
    # calls within the pinned sizes work, and the graph still replays correctly
    b0 = rhs(shape, cplx, 4)
    x0 = h.solve_scaled(b0)
    V = np.asarray(values(rp, ci, v2, batched, 5))
    b = rhs(shape, cplx, 6)
    sv.copy_(cuda(V))
    sb.copy_(cuda(b))
    g.replay()
    torch.cuda.synchronize()
    x = sx.cpu().numpy()
    assert (info.cpu().numpy() == 0).all()
    for j in range(B if batched else 1):
        Vj, xj, bj = (V[j], x[j], b[j]) if batched else (V, x, b)
        assert residual(matrix(rp, ci, Vj, n), xj, bj) <= RES_TOL, j
    V4 = np.asarray(values(rp, ci, v2, batched, 4))
    for j in range(B if batched else 1):
        Vj, xj, bj = (V4[j], x0[j], b0[j]) if batched else (V4, x0, b0)
        assert residual(matrix(rp, ci, Vj, n), xj, bj) <= RES_TOL, j
    del g
    h.close()


# ---- 6. argument refusals ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
def test_argument_refusals(cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("kkt", cplx)
    n, perm_r, perm = prob.n, prs[0], prob.perm
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="factor_device before a successful"):
        h.factor_device()
    h.fill_csr_scaled(rp, ci, v1, perm, perm_r, R0, C0)
    host = np.zeros(1, np.int32)
    with pytest.raises(RuntimeError, match="info must point at device or managed memory"):
        capi._check(capi._fn("factor_device", cplx)(h.h, host.ctypes.data_as(C.c_void_p), stream_ptr()))
    with pytest.raises(RuntimeError, match="batch_factor_device on an unbatched handle"):
        capi._check(capi._fn("batch_factor_device", cplx)(h.h, C.c_void_p(torch.zeros(1, dtype=torch.int32, device="cuda").data_ptr()),
                                                          stream_ptr()))
    assert int(h.factor_device().item()) == 0          # the refused calls left the handle as it was
    h.close()
    bh = capi.BatchHandle(prob, 2)
    with pytest.raises(RuntimeError, match="batch_factor_device before a successful"):
        bh.factor_device()
    bh.close()
    prp, pci, pv = hostlib.row_permute(rp, ci, v1, perm_r)
    sperm = hostlib.schur_order(prp, pci, np.arange(n - 8, n))
    sprob = LUProblem.from_matrix(prp, pci, np.abs(pv), sperm, relax=8, maxsup=32, nschur=8)
    if cplx:
        sprob.dtype = np.dtype(np.complex128)
        for lay in sprob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    sh = capi.SchurHandle(sprob, 8)
    with pytest.raises(RuntimeError, match="Schur handle"):
        sh.factor_device()
    sh.close()


# ---- 7. host state after replays -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx,batched", [(False, False), (True, True)], ids=["d-B1", "z-B4"])
def test_host_state_follows_replays(cplx, batched):
    """selinv's inverse goes with a replayed factorization; a zero pivot the host saw in one replay does not stop the device
    solves after a later good replay; stats() while the capture is open does not wait and leaves the capture valid"""
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("matgen", cplx)
    n = prob.n
    h = handle(prob, batched)
    h.fill_csr_scaled(rp, ci, values(rp, ci, v1, batched, 3), prob.perm, prs[0], R0, C0)
    shape = (B, n) if batched else (n,)
    sv, sb = cuda(values(rp, ci, v2, batched, 4)), cuda(rhs(shape, cplx, 1))
    info = torch.zeros((B,) if batched else (1,), dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        h.refill(sv)
        h.factor_device(info)
        h.solve_scaled(sb)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        h.refill(sv)
        h.factor_device(info)
        h.stats()
        sx = h.solve_scaled(sb)

    def replay(V, b):
        sv.copy_(cuda(V))
        sb.copy_(cuda(b))
        g.replay()
        torch.cuda.synchronize()
        return sx.cpu().numpy()

    def check(V, b, x):
        for j in range(B if batched else 1):
            Vj, xj, bj = (V[j], x[j], b[j]) if batched else (V, x, b)
            assert residual(matrix(rp, ci, Vj, n), xj, bj) <= RES_TOL, j

    V, b = np.asarray(values(rp, ci, v2, batched, 5)), rhs(shape, cplx, 2)
    check(V, b, replay(V, b))
    h.selinv()
    d0 = h.inv_diag()
    V = V * 1.5
    replay(V, b)
    with pytest.raises(RuntimeError, match="selinv on the current factors first"):
        h.inv_diag()
    h.selinv()
    assert rel(h.inv_diag(), d0 / 1.5) <= 1e-12
    # a replay with a zero pivot, seen by a host call; then a good replay: the device solves take its factors
    bad = np.array(V)
    W = np.atleast_2d(bad)
    W[0, rp[n // 3]:rp[n // 3 + 1]] = 0
    x = replay(W if batched else W[0], b)
    assert np.isnan(np.atleast_2d(x)[0]).all() and int(info.cpu().numpy()[0]) > 0
    with pytest.raises(RuntimeError, match="zero pivot|needs a successful"):
        h.logdet()
    replay(V, b)
    b2 = rhs(shape, cplx, 3)
    check(V, b2, h.solve_scaled(cuda(b2)).cpu().numpy())
    del g
    h.close()
