"""The handle's state across a fill that fails, double and doublecomplex: after fill_csr, batch_fill_csr, batch_fill_affine,
fill_csr_scaled or batch_fill_csr_scaled reports entries with no slot, every call that reads the factors refuses, factor
refuses until a new fill, and a good fill and factorization bring the handle back.  And every entry point refused on the
wrong handle kind, or on a Schur handle where it needs complete factors, names itself at the start of its message."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from superlu_dist_b200 import capi
from test_gpu_schur import make as schur_make
from test_scaled_parity import make_problem, panel_coords
from util import poisson_problem

pytestmark = pytest.mark.gpu
KW = dict(N=6, leaf=4, relax=4, maxsup=8)
B = 2
DTYPES = pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
FILLS = ["fill_csr", "batch_fill_csr", "batch_fill_affine", "fill_csr_scaled", "batch_fill_csr_scaled"]


def values(complex_):
    _, (rp, ci, v) = poisson_problem(**KW)
    return rp, ci, v * (1.0 + 0.25j) if complex_ else v


def no_slot(prob, perm):
    """a matrix of one entry, (0, c0), whose permuted position (perm[0], perm[c0]) is not stored in L + U: every index is
    valid, so the fill kernel counts it and reads nothing out of range"""
    lrow, lcol, urow, ucol = panel_coords(prob, prob.layers[0])
    slots = set(zip(lrow.tolist(), lcol.tolist())) | set(zip(urow[urow >= 0].tolist(), ucol[urow >= 0].tolist()))
    c0 = next(c for c in range(prob.n) if (perm[0], perm[c]) not in slots)
    return np.array([0] + [1] * prob.n, np.int32), np.array([c0], np.int32)


@DTYPES
@pytest.mark.parametrize("fill", FILLS)
def test_failed_fill_leaves_no_factors(fill, complex_):
    rp, ci, v = values(complex_)
    prob = make_problem(KW, v)
    n, perm = prob.n, np.asarray(prob.perm, np.int32)
    batched, scaled = fill.startswith("batch"), fill.endswith("scaled")
    h = capi.BatchHandle(prob, B) if batched else capi.Handle(prob, 0)

    def do_fill(rp_, ci_, vals):                           # vals: member 0's values; member j gets (j + 1) vals
        if fill == "batch_fill_affine":
            h.fill_affine(rp_, ci_, vals[None], np.arange(1.0, B + 1)[:, None].astype(v.dtype), perm)
        else:
            vals = np.stack([(j + 1) * vals for j in range(B)]) if batched else vals
            (h.fill_csr_scaled(rp_, ci_, vals, perm, equil=False) if scaled else h.fill_csr(rp_, ci_, vals, perm))

    b = np.ones((B, n) if batched else n, v.dtype)
    do_fill(rp, ci, v)
    assert not np.any(h.factor())
    x0 = h.solve_scaled(b) if scaled else h.solve(b)
    h.selinv()
    rp1, ci1 = no_slot(prob, perm)
    with pytest.raises(RuntimeError, match="no slot"):
        do_fill(rp1, ci1, np.ones(1, v.dtype))
    # the arena holds the half-scattered bad matrix: nothing may read it as factors
    reads = [lambda: h.solve(b), lambda: h.solve(b, trans="T"), lambda: h.rcond(1.0), lambda: h.selinv(), lambda: h.inv_diag(),
             lambda: h.logdet(), lambda: h.inertia()]
    for call in reads:
        with pytest.raises(RuntimeError, match="needs a .*batch_factor" if batched else "needs a successful"):
            call()
    if scaled:
        for call in (lambda: h.solve_scaled(b), lambda: h.refine(b, x0)):
            with pytest.raises(RuntimeError, match="scaled fill"):
                call()
    with pytest.raises(RuntimeError, match="before a successful"):
        h.factor()
    # a good fill and factorization bring the handle back
    do_fill(rp, ci, v)
    assert not np.any(h.factor())
    x = h.solve_scaled(b) if scaled else h.solve(b)
    A = sp.csr_matrix((v, ci, rp), shape=(n, n)).tocoo()
    p = np.arange(n) if scaled else perm                  # solve_scaled works in A's ordering, solve in that of P A P^T
    F = sp.csr_matrix((A.data, (p[A.row], p[A.col])), shape=(n, n))
    for j in range(B if batched else 1):
        xj, bj = (x[j], b[j]) if batched else (x, b)
        assert np.abs((j + 1) * (F @ xj) - bj).max() <= 1e-12 * np.abs(bj).max(), j
    h.close()


def _calls(pre, n, X, I):
    """name -> the arguments after the handle of every entry point that checks the handle (X: a value, vector or output
    buffer, I: an index buffer, both large enough for any of them)"""
    info, la, dfc = C.c_int(), C.c_double(), C.c_double()
    unbatched = {
        "upload": (), "download": (), "factor": (C.byref(info),), "factor_host": (C.byref(info),), "fill_csr": (n, I, I, X, I),
        "solve": (X, n, 1), "solve_trans": (X, n, 1, 1), "gscon": (b"1", 1.0, C.byref(la)), "selinv": (X,),
        "selinv_get": (n, I, I, I, X), "logdet": (C.byref(la), X), "inertia": (X, C.byref(dfc)), "schur_get": (X, n),
        "schur_condense": (X, n, 1), "schur_expand": (X, n, 1), "fill_csr_scaled": (n, I, I, X, I, I, X, X, 0, X),
        "get_scaling": (I, X, X), "solve_scaled": (X, n, 1, 0), "gsrfs": (X, n, X, n, 1, X, None, None),
    }
    batched = {
        "batch_fill_csr": (n, I, I, X, I), "batch_fill_affine": (n, I, I, 1, X, X, I), "batch_factor": (I,),
        "batch_download": (0,), "batch_solve": (X, n, 1), "batch_solve_trans": (X, n, 1, 1), "batch_gscon": (b"1", X, X),
        "batch_selinv": (X,), "batch_selinv_get": (n, I, I, I, X), "batch_logdet": (X, X), "batch_inertia": (X, X),
        "batch_schur_get": (X, n), "batch_schur_condense": (X, n, 1), "batch_schur_expand": (X, n, 1),
        "batch_fill_csr_scaled": (n, I, I, X, I, I, X, X, 0, 0, X), "batch_get_scaling": (0, X, X),
        "batch_solve_scaled": (X, n, 1, 0), "batch_gsrfs": (X, n, X, n, 1, X, None, None),
    }
    named = lambda d: {pre + k: a for k, a in d.items()}  # noqa: E731
    unbatched = named(unbatched)
    if pre == "slu_b200_":
        unbatched.update({"slu_b200_k_level_export": (0, None, 0, None, 0), "slu_b200_k_rerun_schur": (0, 1, C.byref(C.c_float()))})
    return unbatched, named(batched)


# the calls that need complete factors, which a Schur handle of their kind refuses
NOT_ON_SCHUR = {"factor_host", "solve", "solve_trans", "gscon", "selinv", "selinv_get", "logdet", "inertia", "fill_csr_scaled",
                "get_scaling", "solve_scaled", "gsrfs", "k_level_export", "k_rerun_schur"}


@DTYPES
def test_refusals_name_the_call(complex_):
    L = capi.lib()
    pre = "slu_b200_z_" if complex_ else "slu_b200_"
    dt = np.complex128 if complex_ else np.float64
    _, _, v = values(complex_)
    prob = make_problem(KW, v)
    sprob, _, s, _ = schur_make("p8_top", dt)
    n = max(prob.n, sprob.n)
    buf = np.zeros(4 * B * n * n)
    idx = np.zeros(4 * B * n * n, np.int32)
    unbatched, batched = _calls(pre, prob.n, buf.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p))
    h, bh = capi.Handle(prob, 0), capi.BatchHandle(prob, B)
    sh, bsh = capi.SchurHandle(sprob, s), capi.BatchSchurHandle(sprob, B, s)

    def refused(handle, name, want):
        assert getattr(L, name)(handle.h, *(unbatched | batched)[name]) < 0, name
        err = L.slu_b200_last_error()
        assert err.startswith(name.encode()) and any(w in err for w in want), (name, err)

    for name in unbatched:
        refused(bh, name, (b"on a batched handle", b"needs a Schur handle"))
        if name[len(pre):] in NOT_ON_SCHUR:
            refused(sh, name, (b"on a Schur handle",))
    for name in batched:
        refused(h, name, (b"on an unbatched handle",))
        refused(sh, name, (b"on an unbatched handle",))
        if name[len(pre + "batch_"):] in NOT_ON_SCHUR:
            refused(bsh, name, (b"on a Schur handle",))
    for handle in (h, bh, sh, bsh):
        handle.close()
