"""Batched doublecomplex handles (slu_b200_z_batch_*): B complex matrices of one sparsity pattern factored and solved
together on one shared analysis -- the frequency-sweep workload (K - w^2 M + i w C at many w).  Every member must match
the oracle's complex factors of its own values; the batch must take exactly the launches of one unbatched complex
factorization; a zero or tiny pivot stays in its member; misuse fails loudly and names the z calls."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi, hostlib, matgen
from test_gpu_solve_complex import complex_csr
from util import complex_problem, poisson_problem, rel_err

gpu = pytest.mark.gpu
TOL = 1e-10
B = 5
CASES = [dict(N=12, leaf=16, relax=16, maxsup=128), dict(N=6, leaf=4, relax=8, maxsup=200, fem=3),
         dict(N=16, leaf=16, relax=32, maxsup=256)]   # the top separator is one 256-column supernode


def members(kw, batch=B, seed=0):
    """The CSR pattern and the (batch, nnz) complex128 member values: complex_csr's matrix (complex off-diagonals)
    scaled per member by matgen.batch_values."""
    rp, ci, v = complex_csr(**kw)
    return rp, ci, matgen.batch_values(rp, ci, v, batch, seed)


def member_problem(kw, rp, ci, vals, tiny=None):
    """An unfactored complex128 problem holding one member's values, assembled as util.complex_problem does (fill_layer
    is real-only): one problem filled with the real parts, one with the imaginary parts, combined.  tiny = thresh turns
    on tiny-pivot replacement (options and oracle)."""
    re, _ = poisson_problem(**kw)
    im, _ = poisson_problem(**kw)
    re.fill_layer(0, rp, ci, np.ascontiguousarray(vals.real))
    im.fill_layer(0, rp, ci, np.ascontiguousarray(vals.imag))
    re.dtype = np.dtype(np.complex128)
    lay = re.layers[0]
    lay.lval = lay.lval.astype(np.complex128) + 1j * im.layers[0].lval
    lay.uval = lay.uval.astype(np.complex128) + 1j * im.layers[0].uval
    if tiny is not None:
        re.replace_tiny_pivot, re.thresh = 1, tiny
    return re


def factor_batch(prob, rp, ci, vals, **opt):
    h = capi.BatchHandle(prob, len(vals), **opt)
    h.fill_csr(rp, ci, vals, prob.perm)
    return h, h.factor()


def assert_matches_oracle(prob, kw, rp, ci, vals_j, tiny=None):
    chk = member_problem(kw, rp, ci, vals_j, tiny)
    oinfo, _, _ = oracle.factor(chk)
    assert oinfo == 0
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL


def _crandn(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def test_batch_values_complex():
    """CPU: complex members take the float64 members' real scale factors, on both parts."""
    rp, ci, v = hostlib.poisson3d(4)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    vz = v + 1j * np.where(rows == ci, 0.5 * v, 0.25)
    real = matgen.batch_values(rp, ci, v, 6, seed=7)
    z = matgen.batch_values(rp, ci, vz, 6, seed=7)
    assert real.dtype == np.float64 and z.dtype == np.complex128 and z.shape == real.shape == (6, len(v))
    assert np.array_equal(z.real, real)                  # same real part, same seed: the float64 result
    assert np.array_equal(z.imag, matgen.batch_values(rp, ci, vz.imag, 6, seed=7))


@gpu
@pytest.mark.parametrize("kw", CASES)
def test_members_match_oracle(kw):
    rp, ci, vals = members(kw)
    prob = member_problem(kw, rp, ci, vals[0])
    if kw["maxsup"] == 256:
        assert np.diff(np.asarray(prob.xsup)).max() == 256      # the widest complex supernode
    h, info = factor_batch(prob, rp, ci, vals)
    assert info.dtype == np.int32 and info.shape == (B,) and not info.any(), info
    for j in range(B):
        h.download(j)
        assert_matches_oracle(prob, kw, rp, ci, vals[j])
    st = h.stats()
    assert st.reserved[1] == 0 and st.t_factor_s > 0
    h.close()


@gpu
def test_batch_of_one_matches_unbatched_handle():
    kw = CASES[0]
    rp, ci, vals = members(kw, batch=1, seed=3)
    prob = member_problem(kw, rp, ci, vals[0])
    h, info = factor_batch(prob, rp, ci, vals)
    assert info.tolist() == [0]
    h.download(0)
    got = prob.layers[0].copy()
    h.close()
    ref = member_problem(kw, rp, ci, vals[0])
    u = capi.Handle(ref, 0)
    u.fill_csr(rp, ci, vals[0], ref.perm)
    assert u.factor() == 0
    u.download()
    u.close()
    assert rel_err(got.lval, ref.layers[0].lval) <= 1e-13 and rel_err(got.uval, ref.layers[0].uval) <= 1e-13


@gpu
@pytest.mark.parametrize("kw", [CASES[0], CASES[2]])
def test_launches_and_stats_scale(kw):
    rp, ci, vals = members(kw, batch=1)
    prob = member_problem(kw, rp, ci, vals[0])
    u = capi.Handle(prob, 0)
    u.fill_csr(rp, ci, vals[0], prob.perm)
    assert u.factor() == 0
    one = u.stats()
    u.close()
    for batch in (1, 3, 8):
        rp, ci, vals = members(kw, batch=batch)
        h, info = factor_batch(prob, rp, ci, vals)
        assert not info.any()
        st = h.stats()
        h.close()
        assert st.gpu_launches == one.gpu_launches, (batch, st.gpu_launches, one.gpu_launches)
        assert st.ops_fact == batch * one.ops_fact and st.ops_schur == batch * one.ops_schur
        assert st.nnz_l == batch * one.nnz_l and st.nnz_u == batch * one.nnz_u
        assert st.lu_device_bytes == batch * one.lu_device_bytes and st.nlevels == one.nlevels


@gpu
@pytest.mark.parametrize("kw", [CASES[0], CASES[1]])
def test_solve(kw):
    rp, ci, vals = members(kw)
    mats = [member_problem(kw, rp, ci, vals[j]) for j in range(B)]
    prob = mats[0]
    xtrue = _crandn(np.random.default_rng(2), (B, 3, prob.n))
    b = np.stack([(m.dense(m.layers[0], False) @ xtrue[j].T).T for j, m in enumerate(mats)])
    h = capi.BatchHandle(prob, B)
    h.fill_csr(rp, ci, vals, prob.perm)
    with pytest.raises(RuntimeError, match="slu_b200_z_batch_factor"):
        h.solve(b)                                   # filled, not factored
    assert not h.factor().any()
    for _ in range(2):                               # two solves on one handle
        for rhs, ref in ((b, xtrue), (b[:, 0], xtrue[:, 0])):
            x = h.solve(rhs)
            assert x.dtype == np.complex128 and x.shape == rhs.shape
            for j in range(B):
                assert np.abs(x[j] - ref[j]).max() <= 1e-10 * np.abs(ref[j]).max(), j
    assert h.stats().reserved[4] > 0 and h.stats().reserved[5] > 0
    h.close()


@gpu
def test_zero_pivot_in_one_member():
    kw = CASES[0]
    rp, ci, vals = members(kw)
    prob = member_problem(kw, rp, ci, vals[0])
    perm = np.asarray(prob.perm)
    vals[3][perm[ci] == 0] = 0.0                     # column 1 of P A_3 P^T is 0 + 0i: exact zero pivot there
    h, info = factor_batch(prob, rp, ci, vals)
    assert info.tolist() == [0, 0, 0, 1, 0], info
    for j in (0, 1, 2, 4):
        h.download(j)
        assert_matches_oracle(prob, kw, rp, ci, vals[j])
    with pytest.raises(RuntimeError, match="member 3"):
        h.solve(np.ones((B, prob.n), np.complex128))
    h.close()


@gpu
def test_tiny_pivot_in_one_member():
    """pzgstrf2.c's rule: a pivot with both parts non-zero and |re| + |im| < thresh becomes thresh + 0i, counted once."""
    kw, thresh, m = CASES[0], 1e-2, 2
    rp, ci, vals = members(kw)
    prob = member_problem(kw, rp, ci, vals[0], tiny=thresh)
    perm = np.asarray(prob.perm)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    first = (perm[rows] == 0) & (perm[ci] == 0)      # the first pivot of P A_m P^T
    assert first.sum() == 1
    vals[m][first] = 3e-3 + 4e-3j
    h, info = factor_batch(prob, rp, ci, vals)
    assert not info.any(), info
    assert h.stats().tiny_pivots == 1
    for j in (m, 0):
        h.download(j)
        assert_matches_oracle(prob, kw, rp, ci, vals[j], tiny=thresh)
    h.close()


@gpu
def test_errors():
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    rp, ci, vals = members(kw, batch=2)
    prob = member_problem(kw, rp, ci, vals[0])
    L = capi.lib()
    info = C.c_int(0)
    x = np.ones(prob.n, np.complex128)
    xp = x.ctypes.data_as(C.c_void_p)
    rpp, cip, vp, pp = (np.ascontiguousarray(a).ctypes.data_as(C.c_void_p) for a in
                        (rp, ci, vals[0], np.asarray(prob.perm, np.int32)))
    bh = capi.BatchHandle(prob, 2)
    with pytest.raises(RuntimeError, match="slu_b200_z_batch_fill_csr"):
        bh.factor()                                  # factor before fill
    for rc in (L.slu_b200_z_upload(bh.h), L.slu_b200_z_factor(bh.h, C.byref(info)),
               L.slu_b200_z_factor_host(bh.h, C.byref(info)), L.slu_b200_z_download(bh.h),
               L.slu_b200_z_fill_csr(bh.h, prob.n, rpp, cip, vp, pp), L.slu_b200_z_solve(bh.h, xp, prob.n, 1)):
        assert rc < 0
        err = L.slu_b200_last_error()
        assert b"batched handle" in err and err.startswith(b"slu_b200_z_") and b"slu_b200_z_batch_*" in err, err
    with pytest.raises(RuntimeError, match="matrix order"):
        bh.fill_csr(rp[:-1], ci, vals, prob.perm)    # wrong n
    with pytest.raises(ValueError, match="vals must have shape"):
        bh.fill_csr(rp, ci, vals[:1], prob.perm)     # one member's values for a batch of two
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    for m in (-1, 2):
        with pytest.raises(RuntimeError, match="slu_b200_z_batch_download: member .* out of range"):
            bh.download(m)
    bh.close()
    h = capi.Handle(prob, 0)
    ib = np.zeros(2, np.int32).ctypes.data_as(C.c_void_p)
    for rc in (L.slu_b200_z_batch_fill_csr(h.h, prob.n, rpp, cip, vp, pp), L.slu_b200_z_batch_factor(h.h, ib),
               L.slu_b200_z_batch_solve(h.h, xp, prob.n, 1), L.slu_b200_z_batch_download(h.h, 0)):
        assert rc < 0
        err = L.slu_b200_last_error()
        assert b"unbatched handle" in err and err.startswith(b"slu_b200_z_batch_"), err
    h.close()
    with pytest.raises(RuntimeError, match="slu_b200_z_batch_create: batch = 0"):
        capi.BatchHandle(prob, 0)
    wide = complex_problem(npdep=2, **kw)
    with pytest.raises(RuntimeError, match="1 x 1 x 1"):
        capi.BatchHandle(wide, 2)
    with pytest.raises(RuntimeError, match="single-GPU"):
        capi.BatchHandle(prob, 2, world_size=2)
