"""Iterative refinement and condition estimation on the caller's CUDA stream: slu_b200_gsrfs_device, _gscon_device, their
batched and doublecomplex twins, through Handle / BatchHandle.refine and .rcond with torch CUDA tensors and through the raw C
calls.  The device loops against the host loops (gsrfs, gscon) and the NumPy / SciPy restatements; refinement steps taken on
the device; no host wait; one CUDA graph of refill -> factor_device -> solve_scaled_device -> gsrfs_device -> gscon_device
replayed with value sets that need different step counts; a member with a zero pivot; the refusals."""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from superlu_dist_b200 import LUProblem, capi, hostlib
from test_gpu_device_io import SLEEP_CYCLES, members, rhs, setup, stream_ptr
from test_gpu_refine import DENSE_MAX, abs1, ferr_weights, lacn2, numpy_berr, residual_rows, true_forward_error
from test_static_pivot_cpu import csr_parts, kkt

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
B = 4
BERR_TOL = 1e-14
X_TOL = 1e-14
FERR_TOL = 1e-10
RCOND_TOL = 1e-12
CASES = [(name, cplx, batched) for name in ("matgen", "kkt") for cplx in (False, True) for batched in (False, True)]
IDS = [f"{n}-{'z' if c else 'd'}-{'B4' if b else 'B1'}" for n, c, b in CASES]


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return None if t is None else t.cpu().numpy()


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def handle(prob, batched):
    return capi.BatchHandle(prob, B) if batched else capi.Handle(prob, 0)


def prepared(name, cplx, batched, seed=3):
    """a handle after the scaled fill of setup()'s matrix (B value sets when batched) and a successful factor"""
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    V = members(rp, ci, v1, seed) if batched else v1
    h = handle(prob, batched)
    h.fill_csr_scaled(rp, ci, V, prob.perm, prs[0], R0, C0)
    assert (np.atleast_1d(h.factor()) == 0).all()
    return h, prob, rp, ci, V, prs, R0, C0


def per_member(a, batched):
    """(members, ...) view of a batched or unbatched array"""
    return a if batched else a[None]


def check_refinement(rp, ci, V, b, xd, berr, steps, ferr, batched, ref=None, name="", ferr_tol=FERR_TOL):
    """berr = the NumPy restatement on the returned x, bit for bit; ferr against lacn2 driven by SciPy (and at least the true
    forward error for n <= DENSE_MAX); ref = (x, berr, steps) of the host loop: x to X_TOL, steps equal or one apart with both
    berr <= BERR_TOL.  ferr_tol: where pivots were replaced, the estimate solves with those factors and the reference with
    SciPy's LU of A, so the two operators differ by the replacement"""
    n = b.shape[-1]
    cplx = np.iscomplexobj(b)
    Vm, bm, xm, bem, stm = (per_member(np.asarray(a), batched) for a in (V, b, xd, berr, steps))
    fem = None if ferr is None else per_member(ferr, batched)
    if ref is not None:
        assert rel(xd, ref[0]) <= X_TOL, (name, rel(xd, ref[0]))
        for bd, bh, sd, sh in zip(bem.ravel(), per_member(ref[1], batched).ravel(), stm.ravel(), per_member(ref[2], batched).ravel()):
            assert sd == sh or (abs(int(sd) - int(sh)) == 1 and bd <= BERR_TOL and bh <= BERR_TOL), (name, sd, sh, bd, bh)
    for j in range(Vm.shape[0]):
        A = sp.csr_matrix((Vm[j], ci, rp), shape=(n, n))
        lu = spl.splu(A.tocsc()) if fem is not None else None
        for k in range(bm.shape[1]):
            assert bem[j, k] == numpy_berr(rp, ci, Vm[j], xm[j, k], bm[j, k]), (name, j, k)
            assert bem[j, k] <= BERR_TOL and 0 <= stm[j, k] <= 20, (name, j, k, bem[j, k])
            if fem is None:
                continue
            W = ferr_weights(*residual_rows(rp, ci, Vm[j], xm[j, k], bm[j, k]))
            est, _ = lacn2(lambda t: W * lu.solve(t, trans="H" if cplx else "T"), lambda t: lu.solve(W * t), n, cplx)
            fref = est / abs1(xm[j, k]).max()
            assert abs(fem[j, k] - fref) <= ferr_tol * fref, (name, j, k, fem[j, k], fref)
            if n <= DENSE_MAX:
                assert fem[j, k] >= true_forward_error(A, xm[j, k], bm[j, k]), (name, j, k)


# ---- 1. the device loops compute what the host loops compute -------------------------------------------------------------
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
def test_device_matches_host(name, cplx, batched):
    h, prob, rp, ci, V, *_ = prepared(name, cplx, batched)
    n = prob.n
    b = rhs((B, 2, n) if batched else (2, n), cplx, 5)
    x0 = h.solve_scaled(b)
    xh, berr_h, steps_h, ferr_h = h.refine(b, x0)
    xd, berr, steps, ferr = h.refine(cuda(b), cuda(x0))
    assert xd.is_cuda and berr.dtype == torch.float64 and steps.dtype == torch.int32 and ferr.dtype == torch.float64
    assert tuple(berr.shape) == tuple(steps.shape) == tuple(ferr.shape) == b.shape[:-1]
    st = h.stats()
    assert st.reserved[4] == 0 and st.reserved[5] > 0
    check_refinement(rp, ci, V, b, host(xd), host(berr), host(steps), host(ferr), batched, (xh, berr_h, steps_h), name)
    # ferr=False: no estimate, the same refinement
    x2, berr2, _, fe2 = h.refine(cuda(b), cuda(x0), ferr=False)
    assert fe2 is None and rel(host(x2), xh) <= X_TOL
    # one right-hand side per member
    b1 = b[:, 0] if batched else b[0]
    x1, be1, _, _ = h.refine(cuda(b1), cuda(x0[:, 0] if batched else x0[0]))
    assert tuple(be1.shape) == b1.shape[:-1] and rel(host(x1), xh[:, 0] if batched else xh[0]) <= X_TOL
    # the condition estimate, per member, both norms, anorm 0 and +inf -> 0
    anorm = np.array([1.7, 0.0, np.inf, 3.2]) if batched else np.array([1.7])
    for norm in ("1", "I"):
        rd = host(h.rcond(cuda(anorm if batched else anorm[0:1]), norm))
        st = h.stats()
        assert st.reserved[4] == 0 and st.reserved[5] > 0 and st.reserved[6] == 0 and st.reserved[7] == 0
        rh = np.atleast_1d(h.rcond(anorm if batched else anorm[0], norm))
        assert np.allclose(np.atleast_1d(rd), rh, rtol=RCOND_TOL, atol=0), (name, norm, rd, rh)
        if batched:
            assert rd[1] == 0.0 and rd[2] == 0.0 and rd[0] > 0
    if not batched:
        for a in (0.0, np.inf):
            assert float(h.rcond(cuda(np.array([a])))) == 0.0
    h.close()


# ---- 2. the loop iterates on the device ----------------------------------------------------------------------------------
def tiny_pivot_kkt(cplx):
    """KKT [K, B^T; B, D] with the constraints eliminated first and the diagonal of D in the pattern.  values(zero=True):
    D = 1e-20 I, every constraint pivot tiny, replaced by sqrt(eps) ||A|| (solve_scaled's berr ~1e-6, several refinement
    steps); values(zero=False): D = -I, no replacement (0 or 1 step).  -> (prob, rp, ci, values)"""
    A = kkt(16, 40, 3)
    n, m = A.shape[0], 40
    S = sp.csr_matrix(A + sp.diags(np.r_[np.zeros(n - m), np.ones(m)]))
    rp, ci, v = csr_parts(S)
    rows = np.repeat(np.arange(n), np.diff(rp))
    dz = (rows == ci) & (rows >= n - m)
    perm = np.concatenate([np.arange(n - m) + m, np.arange(m)]).astype(np.int32)
    prob = LUProblem.from_matrix(rp, ci, np.abs(v), perm, relax=8, maxsup=32)
    prob.replace_tiny_pivot = 1
    prob.thresh = np.sqrt(np.finfo(np.float64).eps) * abs(A).sum(axis=1).max()
    if cplx:
        prob.dtype = np.dtype(np.complex128)
        for lay in prob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)

    def values(zero, scale=1.0):
        w = np.array(v, np.complex128 if cplx else np.float64) * scale
        w[dz] = 1e-20 if zero else -1.0
        return w * (1.0 + 0.3j) if cplx else w

    return prob, rp, ci, values


@pytest.mark.parametrize("cplx", [False, True])
def test_loop_iterates_on_device(cplx):
    prob, rp, ci, values = tiny_pivot_kkt(cplx)
    n, v = prob.n, values(True)
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v, prob.perm, equil=False)
    assert h.factor() == 0 and h.stats().tiny_pivots > 0
    b = rhs(n, cplx, 1)
    x0 = h.solve_scaled(b)
    before = numpy_berr(rp, ci, v, x0, b)
    assert before > 1e-10
    x, berr, steps, ferr = h.refine(cuda(b), cuda(x0))
    x, berr, steps = host(x), float(berr), int(steps)
    assert steps >= 2 and berr <= BERR_TOL, (steps, berr)
    assert berr == numpy_berr(rp, ci, v, x, b)
    xh, berr_h, steps_h, _ = h.refine(b, x0)
    assert rel(x, xh) <= X_TOL and abs(steps - steps_h) <= 1
    print(f"\ntiny pivots ({'z' if cplx else 'd'}): berr {before:.2e} -> {berr:.2e} in {steps} device steps (host {steps_h})")
    h.close()


# ---- 3. no host wait -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True])
def test_no_host_wait(cplx):
    h, prob, rp, ci, V, *_ = prepared("kkt", cplx, False)
    n = prob.n
    b = rhs((2, n), cplx, 3)
    x0 = h.solve_scaled(b)
    bd, xd, an = cuda(b), cuda(x0), cuda(np.array([2.5]))
    h.refine(bd, xd)                       # the first call allocates and captures its graph
    h.rcond(an, "I")
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    t0 = time.perf_counter()
    x, berr, steps, ferr = h.refine(bd, xd)
    rc = h.rcond(an, "I")
    dt = time.perf_counter() - t0
    pending = not torch.cuda.current_stream().query()
    torch.cuda.synchronize()
    assert pending and dt < 0.01, dt
    xh, berr_h, steps_h, ferr_h = h.refine(b, x0)
    check_refinement(rp, ci, V, b, host(x), host(berr), host(steps), host(ferr), False, (xh, berr_h, steps_h))
    assert np.allclose(float(rc), h.rcond(2.5, "I"), rtol=RCOND_TOL, atol=0)
    h.close()


# ---- 4. one graph, data-dependent step counts ----------------------------------------------------------------------------
def iteration(h, sv, sb, info, anorm):
    h.refill(sv)
    h.factor_device(info)
    sx = h.solve_scaled(sb)
    x, berr, steps, ferr = h.refine(sb, sx)
    return x, berr, steps, ferr, h.rcond(anorm, "1")


@pytest.mark.parametrize("cplx,batched", [(False, False), (True, False), (False, True), (True, True)], ids=["d-B1", "z-B1", "d-B4", "z-B4"])
def test_graph_replay(cplx, batched):
    prob, rp, ci, values = tiny_pivot_kkt(cplx)
    n = prob.n

    def vals(zero):
        if not batched:
            return values(zero)
        return np.stack([values(zero, 1.0 + 0.1 * j) for j in range(B)])

    h, e = handle(prob, batched), handle(prob, batched)
    for x in (h, e):
        x.fill_csr_scaled(rp, ci, vals(False), prob.perm, equil=False)
    shape = (B, n) if batched else (n,)
    cnt = (B,) if batched else (1,)
    sv, sb = cuda(vals(False)), cuda(rhs(shape, cplx, 1))
    info = torch.zeros(cnt, dtype=torch.int32, device="cuda")
    an = torch.full(cnt, 4.0, dtype=torch.float64, device="cuda")
    side = torch.cuda.Stream()                 # warm-up outside capture: slot map, buffers, side streams
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        iteration(h, sv, sb, info, an)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = iteration(h, sv, sb, info, an)
    seen = []
    for it, zero in enumerate((False, True, False)):
        V, b = vals(zero), rhs(shape, cplx, 10 + it)
        sv.copy_(cuda(V))
        sb.copy_(cuda(b))
        g.replay()
        torch.cuda.synchronize()
        x, berr, steps, ferr, rc = (host(t) for t in out)
        assert (host(info) == 0).all()
        ref = [host(t) for t in iteration(e, cuda(V), cuda(b), torch.zeros_like(info), an)]
        assert rel(x, ref[0]) <= X_TOL, (it, rel(x, ref[0]))
        check_refinement(rp, ci, V, b[..., None, :], x[..., None, :], berr[..., None], steps[..., None], ferr[..., None], batched,
                         name=f"replay {it}", ferr_tol=1e-5 if zero else FERR_TOL)
        assert np.array_equal(steps, ref[2]) or (np.abs(steps - ref[2]).max() <= 1 and (ref[1] <= BERR_TOL).all())
        # with replaced pivots F is ill-conditioned: the two factorizations' last-bit differences move the estimate more
        assert np.allclose(rc, ref[4], rtol=1e-6 if zero else RCOND_TOL, atol=0), (it, rc, ref[4])
        seen.append(int(np.max(steps)))
    assert seen[1] >= 2 and seen[1] > min(seen[0], seen[2]), seen
    print(f"\ngraph replay ({'z' if cplx else 'd'}, {'B4' if batched else 'B1'}): steps per replay {seen}")
    del g
    h.close()
    e.close()


# ---- 5. a member with an exact zero pivot --------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cplx,batched", CASES, ids=IDS)
def test_zero_pivot_member(name, cplx, batched):
    prob, rp, ci, v1, v2, prs, R0, C0 = setup(name, cplx)
    n = prob.n
    bad = 1 if batched else 0
    V1 = members(rp, ci, v1, 3) if batched else v1
    V2 = np.atleast_2d(np.array(members(rp, ci, v2, 4) if batched else v2))
    W = V2.copy()
    row = n // 3                                      # a zero row of A: an exact zero pivot in F
    W[bad, rp[row]:rp[row + 1]] = 0
    if not batched:
        V2, W = V2[0], W[0]
    hd, hg = handle(prob, batched), handle(prob, batched)
    for h in (hd, hg):
        h.fill_csr_scaled(rp, ci, V1, prob.perm, prs[0], R0, C0)
    cnt = (B,) if batched else (1,)
    b = rhs((B, 2, n) if batched else (2, n), cplx, 7)
    an = cuda(np.full(cnt, 3.0))
    res = []
    for h, vals in ((hd, W), (hg, V2)):               # the batch with the zero-pivot member, and one without it
        h.refill(cuda(vals))
        info = h.factor_device()
        x0 = h.solve_scaled(cuda(b))
        x, berr, steps, ferr = h.refine(cuda(b), x0)
        res.append([host(t) for t in (info, x, berr, steps, ferr, h.rcond(an, "1"))])
    (info, x, berr, steps, ferr, rc), good = res
    rc = np.atleast_1d(rc)
    assert info[bad] > 0
    xm, bem, stm, fem = (per_member(a, batched) for a in (x, berr, steps, ferr))
    assert np.isnan(xm[bad].real).all() and np.isnan(bem[bad]).all() and np.isnan(fem[bad]).all() and np.isnan(rc[bad])
    if cplx:
        assert np.isnan(xm[bad].imag).all()
    assert (stm[bad] == 0).all()
    gx, gs, grc = per_member(good[1], batched), per_member(good[3], batched), np.atleast_1d(good[5])
    ok = [j for j in range(B if batched else 1) if j != bad]
    if ok:
        Wm, bm = per_member(W, batched), per_member(b, batched)
        check_refinement(rp, ci, Wm[ok], bm[ok], xm[ok], bem[ok], stm[ok], fem[ok], True, name=name)
    for j in ok:
        assert rel(xm[j], gx[j]) <= X_TOL and np.allclose(rc[j], grc[j], rtol=RCOND_TOL, atol=0), (name, j)
        assert (np.abs(stm[j].astype(int) - gs[j]) <= 1).all(), (name, j)
    hd.close()
    hg.close()


# ---- 6. refusals ---------------------------------------------------------------------------------------------------------
def error_of(call):
    with pytest.raises(RuntimeError) as e:
        call()
    return str(e.value)


@pytest.mark.parametrize("cplx", [False, True])
def test_refusals(cplx):
    h, prob, rp, ci, V, prs, R0, C0 = prepared("kkt", cplx, False)
    n = prob.n
    b = rhs(n, cplx, 2)
    x0 = h.solve_scaled(b)
    bd, xd = cuda(b), cuda(x0)

    def usable(hh=h):
        x, berr, _, _ = hh.refine(bd, xd)
        assert float(berr) <= BERR_TOL and float(berr) == numpy_berr(rp, ci, V, host(x), b)
        return x

    # under capture: the first call, then a larger nrhs; nothing is enqueued and the capture stays valid
    torch.cuda.synchronize()
    for first in (True, False):
        bb = bd if first else cuda(rhs((3, n), cplx, 4))
        xx = xd if first else torch.zeros_like(bb)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            assert "would allocate device buffers while the stream is capturing" in error_of(lambda: h.refine(bb, xx))
            sy = bd * 2
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(host(sy), 2 * b)
        del g
        if first:
            usable()
    # host pointers, null b / x / berr through the raw call
    fn = capi._fn("gsrfs_device", cplx)
    be = torch.zeros(1, dtype=torch.float64, device="cuda")
    hb, hx = np.array(b), np.array(x0)
    assert fn(h.h, capi._ptr(hb), n, C.c_void_p(xd.data_ptr()), n, 1, C.c_void_p(be.data_ptr()), None, None, stream_ptr()) != 0
    assert "b must point at device or managed memory" in capi.lib().slu_b200_last_error().decode()
    assert fn(h.h, C.c_void_p(bd.data_ptr()), n, capi._ptr(hx), n, 1, C.c_void_p(be.data_ptr()), None, None, stream_ptr()) != 0
    assert "x must point at device or managed memory" in capi.lib().slu_b200_last_error().decode()
    for args in ((None, xd, be), (bd, None, be), (bd, xd, None)):
        p = [None if a is None else C.c_void_p(a.data_ptr()) for a in args]
        assert fn(h.h, p[0], n, p[1], n, 1, p[2], None, None, stream_ptr()) != 0
        assert "null argument" in capi.lib().slu_b200_last_error().decode()
    assert np.array_equal(host(xd), x0)
    # a bad norm character
    assert "norm must be '1', 'O' or 'I'" in error_of(lambda: h.rcond(cuda(np.array([1.0])), "X"))
    usable()
    assert np.allclose(float(h.rcond(cuda(np.array([2.0])), "O")), h.rcond(2.0, "O"), rtol=RCOND_TOL, atol=0)
    h.close()
    # an unscaled handle: no gsrfs_device, gscon_device works
    v1 = V
    hp = capi.Handle(prob, 0)
    hp.fill_csr(*hostlib.row_permute(rp, ci, v1, prs[0]), prob.perm)
    assert hp.factor() == 0
    assert "scaled fill" in error_of(lambda: hp.refine(bd, xd))
    assert np.allclose(float(hp.rcond(cuda(np.array([2.0])))), hp.rcond(2.0), rtol=RCOND_TOL, atol=0)
    hp.close()
    # a Schur handle
    prp, pci, pv = hostlib.row_permute(rp, ci, v1, prs[0])
    sperm = hostlib.schur_order(prp, pci, np.arange(n - 8, n))
    sprob = LUProblem.from_matrix(prp, pci, np.abs(pv), sperm, relax=8, maxsup=32, nschur=8)
    if cplx:
        sprob.dtype = np.dtype(np.complex128)
        for lay in sprob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    sh = capi.SchurHandle(sprob, 8)
    assert "Schur handle" in error_of(lambda: sh.refine(bd, xd))
    assert "Schur handle" in error_of(lambda: sh.rcond(cuda(np.array([1.0]))))
    sh.close()
