"""Partial factorization on one GPU (slu_b200_schur_* and the z twins): S = A22 - A21 A11^-1 A12 against a dense NumPy
Schur complement and exactly 0 off the stored pattern, condense / expand against dense partial solves and SciPy's
solution of the whole system, the eliminated panels against a full factorization, determinism, the smaller plan on the
top-separator case, a singular A22 block the partial factorization never pivots on, and every refusal.  The host paths
no other test takes: schur_get and condense / expand into padded host arrays, upload of host panels, and refactoring one
handle with new values."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from superlu_dist_b200 import capi
from test_scaled_parity import mixed_values, panel_coords
from test_schur_symbolic_cpu import CASES, dense_F, schur_problem
from test_unsym_skyline_cpu import fill

pytestmark = pytest.mark.gpu
TOL = 1e-10
DTYPES = [np.float64, np.complex128]


def make(name, dtype, seed=7, dense=True):
    """-> (problem of dtype, (rowptr, colind, values), s, F = P A P^T dense, None unless dense)"""
    prob, (rp, ci, v), schur = schur_problem(name)
    cx = np.dtype(dtype).kind == "c"
    vals = mixed_values(rp, ci, v, seed, cx)
    if cx:
        prob.dtype = np.dtype(np.complex128)
        for lay in prob.layers.values():
            lay.lval = lay.lval.astype(np.complex128)
            lay.uval = lay.uval.astype(np.complex128)
    return prob, (rp, ci, vals), len(schur), dense_F(rp, ci, vals, np.asarray(prob.perm)) if dense else None


def schur_ref(F, n1):
    A11, A12, A21, A22 = F[:n1, :n1], F[:n1, n1:], F[n1:, :n1], F[n1:, n1:]
    return A22 - A21 @ np.linalg.solve(A11, A12)


def stored_mask(prob, n1):
    lrow, lcol, urow, ucol = panel_coords(prob, prob.layers[0])
    u = urow >= 0
    r, c = np.concatenate([lrow, urow[u]]), np.concatenate([lcol, ucol[u]])
    keep = (r >= n1) & (c >= n1)
    m = np.zeros((prob.n - n1,) * 2, bool)
    m[r[keep] - n1, c[keep] - n1] = True
    return m


def factored(prob, rp, ci, vals, s):
    h = capi.SchurHandle(prob, s)
    h.fill_csr(rp, ci, vals, prob.perm)
    assert h.factor() == 0
    return h


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_schur_condense_expand(name, dtype):
    prob, (rp, ci, vals), s, F = make(name, dtype)
    n = prob.n
    n1 = n - s
    h = factored(prob, rp, ci, vals, s)
    S = h.schur()
    Sref = schur_ref(F, n1)
    scale = np.abs(Sref).max()
    assert np.abs(S - Sref).max() <= TOL * scale, np.abs(S - Sref).max() / scale
    assert np.all(S[~stored_mask(prob, n1)] == 0)
    S2 = h.schur()
    assert S.tobytes() == S2.tobytes()                                       # bit-identical
    A = sp.csr_matrix((vals, ci, rp), shape=(n, n))
    perm = np.asarray(prob.perm)
    rng = np.random.default_rng(3)
    for nrhs in (1, 5):
        b = rng.standard_normal((nrhs, n))
        if np.dtype(dtype).kind == "c":
            b = b + 1j * rng.standard_normal((nrhs, n))
        bb = b[0] if nrhs == 1 else b
        y = h.condense(bb).reshape(nrhs, n)
        g_ref = (b[:, n1:].T - F[n1:, :n1] @ np.linalg.solve(F[:n1, :n1], b[:, :n1].T)).T
        assert np.abs(y[:, n1:] - g_ref).max() <= TOL * np.abs(g_ref).max()
        y[:, n1:] = np.linalg.solve(S, y[:, n1:].T).T
        x = h.expand(y[0] if nrhs == 1 else y).reshape(nrhs, n)
        for j in range(nrhs):
            res = np.linalg.norm(F @ x[j] - b[j]) / (np.linalg.norm(F, np.inf) * np.linalg.norm(x[j]) + np.linalg.norm(b[j]))
            assert res <= 1e-12, res
            xs = spla.spsolve(A.tocsc(), b[j][perm])                    # A xs = b in the original ordering
            assert np.abs(x[j][perm] - xs).max() <= TOL * np.abs(xs).max()
    st = h.stats()
    assert st.reserved[4] > 0 and st.reserved[5] > 0 and st.reserved[7] > 0
    h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
@pytest.mark.parametrize("name", ["p8_top", "p8_two", "upwind_small"])
def test_eliminated_panels_match_full_factorization(name, dtype):
    """after download, every panel of an eliminated supernode equals the full factorization's (same structure), and
    the Schur panels hold S"""
    prob, (rp, ci, vals), s, F = make(name, dtype)
    full, _, _, _ = make(name, dtype)
    n1 = prob.n - s
    h = factored(prob, rp, ci, vals, s)
    S = h.schur()
    h.download()
    hf = capi.Handle(full, 0)
    hf.fill_csr(rp, ci, vals, full.perm)
    assert hf.factor() == 0
    hf.download()
    xsup = np.asarray(prob.xsup)
    a, b = prob.layers[0], full.layers[0]
    for kind in ("l", "u"):
        off = getattr(a, kind + "val_off")
        va, vb = getattr(a, kind + "val"), getattr(b, kind + "val")
        k1 = int(np.searchsorted(xsup, n1))                                # first Schur supernode
        e = int(off[k1])
        scale = max(np.abs(vb[:e]).max(), 1e-300)
        assert np.abs(va[:e] - vb[:e]).max() <= 1e-12 * scale
    # the downloaded Schur panels are S
    lrow, lcol, urow, ucol = panel_coords(prob, a)
    m = (lrow >= n1) & (lcol >= n1)
    assert np.array_equal(a.lval[m], S[lrow[m] - n1, lcol[m] - n1])
    m = (urow >= n1) & (ucol >= n1)
    assert np.array_equal(a.uval[m], S[urow[m] - n1, ucol[m] - n1])
    # the top separator: fewer levels and launches than the full factorization, eliminated work only
    st, sf = h.stats(), hf.stats()
    assert st.nlevels < sf.nlevels and st.gpu_launches < sf.gpu_launches
    assert st.ops_fact < sf.ops_fact and st.my_supernodes == int(np.searchsorted(xsup, n1))
    h.close()
    hf.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
def test_zero_schur_block(dtype):
    """A21 = A22 = 0 on the pattern (explicit zeros): the full factorization meets a zero pivot at column n - s + 1, the
    partial one never pivots there and S is exactly 0"""
    prob, (rp, ci, vals), s, _ = make("p8_top", dtype)
    full, _, _, _ = make("p8_top", dtype)
    n1 = prob.n - s
    rows = np.repeat(np.arange(prob.n), np.diff(rp))
    v0 = np.where(np.asarray(prob.perm)[rows] >= n1, 0, vals).astype(vals.dtype)
    hf = capi.Handle(full, 0)
    hf.fill_csr(rp, ci, v0, full.perm)
    assert hf.factor() == n1 + 1
    hf.close()
    h = capi.SchurHandle(prob, s)
    h.fill_csr(rp, ci, v0, prob.perm)
    assert h.factor() == 0
    assert np.all(h.schur() == 0)
    h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
def test_refusals(dtype):
    z = np.dtype(dtype).kind == "c"
    L = capi.lib()
    pre = "slu_b200_z_" if z else "slu_b200_"
    prob, (rp, ci, vals), s, _ = make("p8_top", dtype)
    n = prob.n
    # creation
    for bad in (0, n):
        with pytest.raises(RuntimeError, match="nschur"):
            capi.SchurHandle(prob, bad)
    k = 1 + int(np.argmax(np.diff(np.asarray(prob.xsup)) > 1))         # a supernode of more than one column
    with pytest.raises(RuntimeError, match=f"not a supernode boundary: supernode {k - 1}"):
        capi.SchurHandle(prob, n - int(prob.xsup[k - 1]) - 1)
    if not z:
        with pytest.raises(RuntimeError, match="int8"):
            capi.SchurHandle(prob, s, tc_slices=7)
    # before factor
    h = capi.SchurHandle(prob, s)
    with pytest.raises(RuntimeError, match="needs a successful"):
        h.schur()
    with pytest.raises(RuntimeError, match="needs a successful"):
        h.condense(np.ones(n))
    h.fill_csr(rp, ci, vals, prob.perm)
    assert h.factor() == 0
    S0 = h.schur()
    b = np.ones(n, dtype)
    y0 = h.condense(b)
    # every call that needs complete factors fails with a message and leaves the handle usable
    calls = [lambda: h.factor_host(), lambda: h.solve(b), lambda: h.solve(b, trans="T"), lambda: h.rcond(1.0),
             lambda: h.selinv(), lambda: h.inv_diag(), lambda: h.logdet()]
    for call in calls:
        with pytest.raises(RuntimeError, match="Schur handle"):
            call()
    x = np.ones(n, dtype)
    assert getattr(L, pre + "batch_solve")(h.h, x.ctypes.data_as(C.c_void_p), n, 1) < 0
    assert b"unbatched handle" in L.slu_b200_last_error()
    if not z:
        assert L.slu_b200_k_level_export(h.h, 0, None, 0, None, 0) < 0 and b"Schur handle" in L.slu_b200_last_error()
        ms = C.c_float()
        assert L.slu_b200_k_rerun_schur(h.h, 0, 1, C.byref(ms)) < 0 and b"Schur handle" in L.slu_b200_last_error()
    out = np.empty((s, s), dtype, order="F")
    assert getattr(L, pre + "schur_get")(h.h, out.ctypes.data_as(C.c_void_p), s - 1) < 0
    assert b"lds" in L.slu_b200_last_error()
    assert np.array_equal(h.schur(), S0)
    # the solve's update scatter accumulates with atomics, whose order is not fixed: equal up to the last bits
    assert np.abs(h.condense(b) - y0).max() <= 1e-14 * np.abs(y0).max()
    h.close()
    # the schur_* calls on an ordinary and on a batched handle
    plain, _, _, _ = make("p8_top", dtype)
    ho = capi.Handle(plain, 0)
    ho.fill_csr(rp, ci, vals, plain.perm)
    assert ho.factor() == 0
    bh = capi.BatchHandle(plain, 2)
    bh.fill_csr(rp, ci, np.stack([vals, vals]), plain.perm)
    assert not bh.factor().any()
    for hh in (ho.h, bh.h):
        assert getattr(L, pre + "schur_get")(hh, out.ctypes.data_as(C.c_void_p), s) < 0
        assert b"needs a Schur handle" in L.slu_b200_last_error()
        for f in ("schur_condense", "schur_expand"):
            assert getattr(L, pre + f)(hh, x.ctypes.data_as(C.c_void_p), n, 1) < 0
            assert b"needs a Schur handle" in L.slu_b200_last_error()
    ho.close()
    bh.close()


# the host paths, on a small case and on one with a 256-row Schur panel
HOST_CASES = ["p8_top", "p16_w256"]


def _sentinel(dtype):
    return np.array(-7.25 + 3.5j if np.dtype(dtype).kind == "c" else -7.25, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
@pytest.mark.parametrize("name", HOST_CASES)
def test_schur_get_padded_lds(name, dtype):
    """lds = s + 3 (a strided device-to-host copy): the s x s block is schur()'s, the padding rows keep their values"""
    prob, (rp, ci, vals), s, _ = make(name, dtype, dense=False)
    h = factored(prob, rp, ci, vals, s)
    S = h.schur()
    lds = s + 3
    out = np.full((s, lds), _sentinel(dtype))          # column-major s x s with leading dimension lds: out[j, i] = S(i, j)
    pre = "slu_b200_z_" if np.dtype(dtype).kind == "c" else "slu_b200_"
    assert getattr(capi.lib(), pre + "schur_get")(h.h, out.ctypes.data_as(C.c_void_p), lds) == 0
    assert np.array_equal(out[:, :s].T, S)
    assert np.all(out[:, s:] == _sentinel(dtype))
    h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
@pytest.mark.parametrize("name", HOST_CASES)
def test_condense_expand_padded_ldx(name, dtype):
    """ldx = n + 5, nrhs = 3: the same result as ldx = n, the padding of every right-hand side untouched"""
    prob, (rp, ci, vals), s, _ = make(name, dtype, dense=False)
    h = factored(prob, rp, ci, vals, s)
    n, nrhs, ldx = prob.n, 3, prob.n + 5
    rng = np.random.default_rng(5)
    b = rng.standard_normal((nrhs, n)).astype(dtype)
    if np.dtype(dtype).kind == "c":
        b = b + 1j * rng.standard_normal((nrhs, n))
    pre = "slu_b200_z_" if np.dtype(dtype).kind == "c" else "slu_b200_"
    for f, x0 in (("condense", b), ("expand", h.condense(b))):
        want = getattr(h, f)(x0)                                             # ldx = n
        buf = np.full((nrhs, ldx), _sentinel(dtype))
        buf[:, :n] = x0
        assert getattr(capi.lib(), pre + "schur_" + f)(h.h, buf.ctypes.data_as(C.c_void_p), ldx, nrhs) == 0
        # the update scatter accumulates with atomics, whose order is not fixed: equal up to the last bits
        assert np.abs(buf[:, :n] - want).max() <= 1e-14 * np.abs(want).max(), f
        assert np.all(buf[:, n:] == _sentinel(dtype)), f
    h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
@pytest.mark.parametrize("name", HOST_CASES)
def test_upload_host_panels(name, dtype):
    """upload() of panels filled on the host (a complex matrix part by part), then factor(): fill_csr's S"""
    prob, (rp, ci, vals), s, _ = make(name, dtype, dense=False)
    h0 = factored(prob, rp, ci, vals, s)
    S0 = h0.schur()
    h0.close()
    fill(prob, rp, ci, vals)             # before the handle: its view points at the layer's arrays
    h = capi.SchurHandle(prob, s)
    h.upload()
    assert h.factor() == 0
    S = h.schur()
    assert np.abs(S - S0).max() <= 1e-13 * np.abs(S0).max()
    h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["d", "z"])
@pytest.mark.parametrize("name", HOST_CASES)
def test_refactor_with_new_values(name, dtype):
    """fill_csr + factor a second time on one handle (the parameter sweep): the S of a fresh handle for the new values,
    nothing left of the first"""
    prob, (rp, ci, v1), s, _ = make(name, dtype, dense=False)
    fresh, _, _, _ = make(name, dtype, dense=False)
    v2 = make(name, dtype, seed=8, dense=False)[1][2]
    h = factored(prob, rp, ci, v1, s)
    S1 = h.schur()
    h.fill_csr(rp, ci, v2, prob.perm)
    assert h.factor() == 0
    S2 = h.schur()
    hf = factored(fresh, rp, ci, v2, s)
    Sf = hf.schur()
    assert np.abs(S2 - Sf).max() <= 1e-13 * np.abs(Sf).max()
    assert np.abs(S2 - S1).max() > 0.1 * np.abs(S1).max()
    h.close()
    hf.close()
