"""Device-resident refill and solves on the caller's CUDA stream: slu_b200_refill, _solve_device, _solve_scaled_device,
their batched and doublecomplex twins, through Handle / BatchHandle with torch CUDA tensors and through the raw C calls.
The refill against a scaled fill of the same values with the kept R and C, bit for bit; the device solves against the host
solves and SciPy; gsrfs after a refill against the NumPy restatement; the refusals; the stream order in both directions."""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.sparse as sp

from superlu_dist_b200 import LUProblem, capi, hostlib, matgen
from test_gpu_static_pivot import arena, complex_kkt, op, residual
from test_refine_cpu import berr_of, residual_rows
from test_static_pivot_cpu import csr_parts, kkt

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
RES_TOL = 1e-14
AGREE_TOL = 1e-14
B = 4


def matgen_matrix(cplx):
    rp, ci, v = hostlib.poisson3d(8)
    if cplx:
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        v = v + 1j * np.where(rows == ci, 0.5, 0.25 * np.random.default_rng(1).uniform(-1, 1, len(v)))
    return sp.csr_matrix((v, ci, rp), shape=(len(rp) - 1,) * 2)


def kkt_matrix(cplx):
    return complex_kkt(12, 30, 4) if cplx else kkt(16, 40, 3)


MATRICES = {"matgen": matgen_matrix, "kkt": kkt_matrix}


def setup(name, cplx, swap=False):
    """(LUProblem, rp, ci, v1, v2, perm_r list, R, C): A's pattern, two value sets (v2 from matgen.batch_values), the
    matching's perm_r and scalings; with swap a second perm_r (adjacent rows exchanged) and a symbolic structure that holds
    the patterns of both row permutations"""
    A = MATRICES[name](cplx)
    rp, ci, v = csr_parts(A)
    perm_r, R, Cs, _ = hostlib.large_diag_perm(rp, ci, v)
    prs = [perm_r]
    pat = sp.csr_matrix(abs(sp.csr_matrix((v, ci, rp), shape=A.shape)))
    Pr = sp.csr_matrix((np.ones(A.shape[0]), (perm_r, np.arange(A.shape[0]))), shape=A.shape)
    U = Pr @ pat
    if swap:
        p2 = perm_r.copy()
        p2[:-1:2], p2[1::2] = perm_r[1::2], perm_r[:-1:2]
        prs.append(p2)
        P2 = sp.csr_matrix((np.ones(A.shape[0]), (p2, np.arange(A.shape[0]))), shape=A.shape)
        U = U + P2 @ pat
    U = sp.csr_matrix(U)
    U.sort_indices()
    urp, uci = U.indptr.astype(np.int32), U.indices.astype(np.int32)
    perm = hostlib.nd_order_graph(urp, uci, leaf=16)
    prob = LUProblem.from_matrix(urp, uci, U.data, perm, relax=8, maxsup=32)
    if cplx:
        prob.dtype = np.dtype(np.complex128)
        for lay in prob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    v2 = matgen.batch_values(rp, ci, v, 1, seed=11)[0]
    return prob, rp, ci, v, v2, prs, R, Cs


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rhs(shape, cplx, seed):
    rng = np.random.default_rng(seed)
    b = rng.standard_normal(shape)
    return b + 1j * rng.standard_normal(shape) if cplx else b


def members(rp, ci, v, seed):
    """B value sets of A's pattern (batch, nnz)"""
    return matgen.batch_values(rp, ci, v, B, seed=seed)


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- 1. the refill is exact ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(MATRICES))
def test_refill_is_the_scaled_fill_bit_for_bit(name, cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx, swap=True)
    h, h2 = capi.Handle(prob, 0), capi.Handle(prob, 0)
    for perm_r in prs:          # the second scaled fill has another row map: the slot map must be rebuilt
        h.fill_csr_scaled(rp, ci, v1, prob.perm, perm_r, R0, C0, equil=True)
        _, R, Cs = h.scaling()
        h.refill(cuda(v2))
        assert h.stats().reserved[5] >= 1 and h.stats().reserved[4] == 0 and h.stats().t_upload_s == 0
        h.download()
        mine = arena(prob)
        h2.fill_csr_scaled(rp, ci, v2, prob.perm, perm_r, R, Cs, equil=False)
        h2.download()
        ref = arena(prob)
        assert np.array_equal(mine[0], ref[0]) and np.array_equal(mine[1], ref[1]), name
        pr2, R2, C2 = h.scaling()           # the scaling is kept, not redone
        assert np.array_equal(pr2, perm_r) and np.array_equal(R2, R) and np.array_equal(C2, Cs)
        h.refill(cuda(v2))                  # the map is reused: one launch
        assert h.stats().reserved[5] == 1
    h.close()
    h2.close()


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(MATRICES))
def test_batched_refill_is_the_scaled_fill_bit_for_bit(name, cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx, swap=True)
    V1, V2 = members(rp, ci, v1, 3), members(rp, ci, v2, 4)
    bh, bh2 = capi.BatchHandle(prob, B), capi.BatchHandle(prob, B)
    for perm_r in prs:
        bh.fill_csr_scaled(rp, ci, V1, prob.perm, perm_r, R0, C0, equil=True)
        RC = [bh.scaling(j) for j in range(B)]
        bh.refill(cuda(V2))
        mine = []
        for j in range(B):
            bh.download(j)
            mine.append(arena(prob))
        bh2.fill_csr_scaled(rp, ci, V2, prob.perm, perm_r, np.stack([r for r, _ in RC]), np.stack([c for _, c in RC]), equil=False)
        for j in range(B):
            bh2.download(j)
            ref = arena(prob)
            assert np.array_equal(mine[j][0], ref[0]) and np.array_equal(mine[j][1], ref[1]), (name, j)
            assert all(np.array_equal(a, b) for a, b in zip(bh.scaling(j), RC[j]))
    bh.close()
    bh2.close()


# ---- 2. and 4. the factors and the kept A are the new matrix's --------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(MATRICES))
def test_factors_and_refinement_follow_the_refill(name, cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    n = prob.n
    A1 = sp.csr_matrix((v1, ci, rp), shape=(n, n))
    A2 = sp.csr_matrix((v2, ci, rp), shape=(n, n))
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v1, prob.perm, prs[0], R0, C0)
    assert h.factor() == 0
    h.refill(cuda(v2))
    assert h.factor() == 0
    b = rhs((2, n), cplx, 5)
    x = h.solve_scaled(cuda(b)).cpu().numpy()
    assert residual(A2, x, b) <= RES_TOL, name
    assert residual(A1, x, b) > 1e3 * RES_TOL
    xr, berr, steps, _ = h.refine(b, x, ferr=False)
    for j in range(2):
        assert berr[j] == berr_of(*residual_rows(rp, ci, v2, xr[j], b[j])), (name, j)
    h.close()
    bh = capi.BatchHandle(prob, B)
    V1, V2 = members(rp, ci, v1, 3), members(rp, ci, v2, 4)
    bh.fill_csr_scaled(rp, ci, V1, prob.perm, prs[0], R0, C0)
    bh.refill(cuda(V2))
    assert (bh.factor() == 0).all()
    bb = rhs((B, 2, n), cplx, 6)
    x = bh.solve_scaled(cuda(bb)).cpu().numpy()
    xr, berr, _, _ = bh.refine(bb, x, ferr=False)
    for j in range(B):
        Aj = sp.csr_matrix((V2[j], ci, rp), shape=(n, n))
        assert residual(Aj, x[j], bb[j]) <= RES_TOL, (name, j)
        for k in range(2):
            assert berr[j, k] == berr_of(*residual_rows(rp, ci, V2[j], xr[j, k], bb[j, k])), (name, j, k)
    bh.close()


# ---- 3. the device solves are the host solves -------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(MATRICES))
def test_device_solves_match_the_host_solves(name, cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    n = prob.n
    A = sp.csr_matrix((v1, ci, rp), shape=(n, n))
    perm_r, perm = prs[0], prob.perm
    rows = np.repeat(np.arange(n), np.diff(rp))
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v1, perm, perm_r, R0, C0)
    assert h.factor() == 0
    _, R, Cs = h.scaling()
    # F = Pc Pr Dr A Dc Pc^T, the matrix of the plain solves
    F = sp.csr_matrix(((R[rows] * v1) * Cs[ci], (perm[perm_r[rows]], perm[ci])), shape=(n, n))
    dt = torch.complex128 if cplx else torch.float64
    for nrhs in (1, 5):
        b = rhs((nrhs, n), cplx, nrhs)
        for trans in ("N", "T", "H"):
            xd = h.solve(cuda(b), trans=trans).cpu().numpy()
            xh = h.solve(b, trans=trans)
            assert rel(xd, xh) <= AGREE_TOL and residual(op(F, trans), xd, b) <= RES_TOL, (name, trans, nrhs)
            xd = h.solve_scaled(cuda(b), trans=trans).cpu().numpy()
            xh = h.solve_scaled(b, trans=trans)
            assert rel(xd, xh) <= AGREE_TOL and residual(op(A, trans), xd, b) <= RES_TOL, (name, trans, nrhs)
            # ldx > n through the raw call: the padding stays as it was
            ldx = n + 7
            pad = torch.full((nrhs, ldx), 3.0, dtype=dt, device="cuda")
            pad[:, :n] = cuda(b)
            for fn, ref in (("solve_device", h.solve(b, trans=trans)), ("solve_scaled_device", xh)):
                x = pad.clone()
                rc = capi._fn(fn, cplx)(h.h, C.c_void_p(x.data_ptr()), ldx, nrhs, capi._TRANS[trans], stream_ptr())
                assert rc == 0, capi.lib().slu_b200_last_error()
                xc = x.cpu().numpy()
                assert rel(xc[:, :n], ref) <= AGREE_TOL and (xc[:, n:] == 3.0).all(), (fn, trans, nrhs)
    h.close()
    bh = capi.BatchHandle(prob, B)
    V = members(rp, ci, v1, 3)
    bh.fill_csr_scaled(rp, ci, V, perm, perm_r, R0, C0)
    assert (bh.factor() == 0).all()
    for nrhs in (1, 5):
        b = rhs((B, nrhs, n), cplx, 10 + nrhs)
        for trans in ("N", "T", "H"):
            for meth in ("solve", "solve_scaled"):
                xd = getattr(bh, meth)(cuda(b), trans=trans).cpu().numpy()
                xh = getattr(bh, meth)(b, trans=trans)
                assert rel(xd, xh) <= AGREE_TOL, (meth, trans, nrhs)
            for j in range(B):
                Aj = sp.csr_matrix((V[j], ci, rp), shape=(n, n))
                assert residual(op(Aj, trans), xd[j], b[j]) <= RES_TOL, (name, j, trans)
            ldx = n + 5
            pad = torch.full((B, nrhs, ldx), -2.0, dtype=dt, device="cuda")
            pad[:, :, :n] = cuda(b)
            rc = capi._fn("batch_solve_scaled_device", cplx)(bh.h, C.c_void_p(pad.data_ptr()), ldx, nrhs, capi._TRANS[trans], stream_ptr())
            assert rc == 0, capi.lib().slu_b200_last_error()
            xc = pad.cpu().numpy()
            assert rel(xc[:, :, :n], xh) <= AGREE_TOL and (xc[:, :, n:] == -2.0).all()
    one = bh.solve(cuda(rhs((B, n), cplx, 3)))
    assert tuple(one.shape) == (B, n) and one.is_cuda
    bh.close()


# ---- 5. refusals --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
def test_refusals(cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("kkt", cplx)
    n, perm_r, perm = prob.n, prs[0], prob.perm
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="refill needs a scaled fill"):
        h.refill(cuda(v2))
    h.fill_csr(*hostlib.row_permute(rp, ci, v1, perm_r), perm)
    with pytest.raises(RuntimeError, match="refill needs a scaled fill"):
        h.refill(cuda(v2))
    h.fill_csr_scaled(rp, ci, v1, perm, perm_r, R0, C0)
    assert h.factor() == 0
    b = rhs(n, cplx, 1)
    x0 = h.solve_scaled(b)
    # host memory in the raw calls: refused before anything is enqueued, the handle keeps its factors
    hv = np.ascontiguousarray(v2)
    hb = np.array(b)
    with pytest.raises(RuntimeError, match="val must point at device or managed memory"):
        capi._check(capi._fn("refill", cplx)(h.h, hv.ctypes.data_as(C.c_void_p), stream_ptr()))
    for fn in ("solve_device", "solve_scaled_device"):
        with pytest.raises(RuntimeError, match="x must point at device or managed memory"):
            capi._check(capi._fn(fn, cplx)(h.h, hb.ctypes.data_as(C.c_void_p), n, 1, 0, stream_ptr()))
    assert np.array_equal(hb, b)
    assert rel(h.solve_scaled(b), x0) <= AGREE_TOL      # the solves add with atomics: equal up to rounding
    h.refill(cuda(v2))
    for call in (lambda: h.solve(cuda(b)), lambda: h.solve_scaled(cuda(b))):
        with pytest.raises(RuntimeError, match="needs a successful"):
            call()
    with pytest.raises(RuntimeError, match="batch_refill on an unbatched handle"):
        capi._check(capi._fn("batch_refill", cplx)(h.h, C.c_void_p(cuda(v2).data_ptr()), stream_ptr()))
    h.close()
    bh = capi.BatchHandle(prob, 2)
    with pytest.raises(RuntimeError, match="batch_refill needs a scaled fill"):
        bh.refill(cuda(np.stack([v2, v2])))
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
        sh.refill(cuda(v2))
    sh.close()


# ---- 6. and 7. stream order, no host wait ---------------------------------------------------------------------------------
SLEEP_CYCLES = 100_000_000       # ~50 ms at the H100's clocks


@pytest.mark.parametrize("cplx", [False, True])
def test_stream_order_and_no_host_wait(cplx):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup("kkt", cplx)
    n = prob.n
    A2 = sp.csr_matrix((v2, ci, rp), shape=(n, n))
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v1, prob.perm, prs[0], R0, C0)
    # the caller overwrites val right after the refill, on the same stream: the factors are of the old values
    v = cuda(v2)
    h.refill(v)
    v.fill_(float("nan"))
    assert h.factor() == 0
    b = rhs((3, n), cplx, 2)
    assert residual(A2, h.solve_scaled(b), b) <= RES_TOL
    # b written on a side stream after a sleep, solved in that stream's context
    side = torch.cuda.Stream()
    src = cuda(b)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        bt = torch.zeros_like(src)
        torch.cuda._sleep(SLEEP_CYCLES)
        bt.copy_(src)
        x = h.solve_scaled(bt)
        y = x * 1                       # read in stream order on the side stream
    side.synchronize()
    assert residual(A2, y.cpu().numpy(), b) <= RES_TOL
    # no host wait: the call returns while the caller's stream still sleeps
    bd = cuda(b)
    h.solve(bd)
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    t0 = time.perf_counter()
    x = h.solve(bd)
    dt = time.perf_counter() - t0
    pending = not torch.cuda.current_stream().query()
    torch.cuda.synchronize()
    assert pending and dt < 0.01, dt
    assert rel(x.cpu().numpy(), h.solve(b)) <= AGREE_TOL
    h.close()
