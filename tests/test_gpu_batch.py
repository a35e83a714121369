"""Batched handles (slu_b200_batch_*): B matrices of one sparsity pattern factored and solved together on one shared
analysis.  Every member must match the oracle's factors of its own values; the batch must take exactly the launches
of one unbatched factorization; a zero pivot stays in its member; misuse fails loudly."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi, matgen
from util import poisson_problem, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10
B = 5
CASES = [dict(N=12, leaf=16, relax=16, maxsup=128), dict(N=6, leaf=4, relax=8, maxsup=200, fem=3),
         dict(N=16, leaf=16, relax=32, maxsup=256)]


def members(kw, batch=B, seed=0):
    """The batched problem (values of member 0 in its layer) and the (batch, nnz) member values."""
    prob, (rp, ci, v) = poisson_problem(**kw)
    return prob, rp, ci, matgen.batch_values(rp, ci, v, batch, seed)


def member_problem(kw, rp, ci, vals):
    """An unfactored problem holding one member's values (same structure: the symbolic phase ignores values)."""
    p, _ = poisson_problem(**kw)
    p.fill_layer(0, rp, ci, vals)
    return p


def factor_batch(prob, rp, ci, vals, **opt):
    h = capi.BatchHandle(prob, len(vals), **opt)
    h.fill_csr(rp, ci, vals, prob.perm)
    return h, h.factor()


@pytest.mark.parametrize("kw", CASES)
def test_members_match_oracle(kw):
    prob, rp, ci, vals = members(kw)
    if kw["maxsup"] == 256:
        assert np.diff(np.asarray(prob.xsup)).max() == 256      # the top separator: one 256-column supernode on DMMA
    h, info = factor_batch(prob, rp, ci, vals)
    assert info.dtype == np.int32 and info.shape == (B,) and not info.any(), info
    for j in range(B):
        h.download(j)
        chk = member_problem(kw, rp, ci, vals[j])
        oinfo, _, _ = oracle.factor(chk)
        assert oinfo == 0
        a, b = prob.layers[0], chk.layers[0]
        assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL, j
    st = h.stats()
    assert st.reserved[1] == 0 and st.t_factor_s > 0
    h.close()


def test_batch_of_one_matches_unbatched_handle():
    kw = CASES[0]
    prob, rp, ci, vals = members(kw, batch=1, seed=3)
    h, info = factor_batch(prob, rp, ci, vals)
    assert info.tolist() == [0]
    h.download(0)
    got = prob.layers[0].copy()
    h.close()
    ref, _ = poisson_problem(**kw)
    u = capi.Handle(ref, 0, tc_slices=-1)
    u.fill_csr(rp, ci, vals[0], ref.perm)
    assert u.factor() == 0
    u.download()
    u.close()
    assert rel_err(got.lval, ref.layers[0].lval) <= 1e-13 and rel_err(got.uval, ref.layers[0].uval) <= 1e-13


@pytest.mark.parametrize("kw", [CASES[0], CASES[2]])
def test_launches_and_stats_scale(kw):
    prob, rp, ci, vals = members(kw, batch=1)
    u = capi.Handle(prob, 0, tc_slices=-1)
    u.fill_csr(rp, ci, vals[0], prob.perm)
    assert u.factor() == 0
    one = u.stats()
    u.close()
    for batch in (1, 3, 8):
        prob, rp, ci, vals = members(kw, batch=batch)
        h, info = factor_batch(prob, rp, ci, vals)
        assert not info.any()
        st = h.stats()
        h.close()
        assert st.gpu_launches == one.gpu_launches, (batch, st.gpu_launches, one.gpu_launches)
        assert st.ops_fact == batch * one.ops_fact and st.ops_schur == batch * one.ops_schur
        assert st.nnz_l == batch * one.nnz_l and st.nnz_u == batch * one.nnz_u
        assert st.lu_device_bytes == batch * one.lu_device_bytes and st.nlevels == one.nlevels


@pytest.mark.parametrize("kw", [CASES[0], CASES[1]])
def test_solve(kw):
    prob, rp, ci, vals = members(kw)
    every = np.ones(prob.nsupers, bool)
    rng = np.random.default_rng(2)
    xtrue = rng.standard_normal((B, 3, prob.n))
    mats = [member_problem(kw, rp, ci, vals[j]) for j in range(B)]
    b = np.stack([m.matvec([(m.layers[0], every)], xtrue[j], 0) for j, m in enumerate(mats)])
    h = capi.BatchHandle(prob, B)
    h.fill_csr(rp, ci, vals, prob.perm)
    with pytest.raises(RuntimeError, match="batch_factor"):
        h.solve(b)                                   # filled, not factored
    assert not h.factor().any()
    for _ in range(2):                               # two solves on one handle
        for rhs, ref in ((b, xtrue), (b[:, 0], xtrue[:, 0])):
            x = h.solve(rhs)
            assert x.shape == rhs.shape
            for j in range(B):
                assert np.abs(x[j] - ref[j]).max() <= 1e-10 * np.abs(ref[j]).max(), j
    assert h.stats().reserved[4] > 0 and h.stats().reserved[5] > 0
    h.close()


def test_zero_pivot_in_one_member():
    kw = CASES[0]
    prob, rp, ci, vals = members(kw)
    perm = np.asarray(prob.perm)
    vals[3][perm[ci] == 0] = 0.0                     # column 1 of P A_3 P^T is zero: exact zero pivot there
    h, info = factor_batch(prob, rp, ci, vals)
    assert info[3] == 1 and not np.delete(info, 3).any(), info
    for j in (0, 1, 2, 4):
        h.download(j)
        chk = member_problem(kw, rp, ci, vals[j])
        oracle.factor(chk)
        assert rel_err(prob.layers[0].lval, chk.layers[0].lval) < TOL and rel_err(prob.layers[0].uval, chk.layers[0].uval) < TOL
    with pytest.raises(RuntimeError, match="member 3"):
        h.solve(np.ones((B, prob.n)))
    h.close()


def test_errors():
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    prob, rp, ci, vals = members(kw, batch=2)
    L = capi.lib()
    info = C.c_int(0)
    x = np.ones(prob.n)
    xp = x.ctypes.data_as(C.c_void_p)
    rpp, cip, vp, pp = (np.ascontiguousarray(a).ctypes.data_as(C.c_void_p) for a in
                        (rp, ci, vals[0], np.asarray(prob.perm, np.int32)))
    bh = capi.BatchHandle(prob, 2)
    with pytest.raises(RuntimeError, match="batch_fill_csr"):
        bh.factor()                                  # factor before fill
    for rc in (L.slu_b200_upload(bh.h), L.slu_b200_factor(bh.h, C.byref(info)), L.slu_b200_factor_host(bh.h, C.byref(info)),
               L.slu_b200_download(bh.h), L.slu_b200_fill_csr(bh.h, prob.n, rpp, cip, vp, pp), L.slu_b200_solve(bh.h, xp, prob.n, 1),
               L.slu_b200_k_level_export(bh.h, 0, None, 0, None, 0), L.slu_b200_k_rerun_schur(bh.h, 0, 1, C.byref(C.c_float()))):
        assert rc < 0
        assert b"batched handle" in L.slu_b200_last_error()
    with pytest.raises(RuntimeError, match="matrix order"):
        bh.fill_csr(rp[:-1], ci, vals, prob.perm)    # wrong n
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    for m in (-1, 2):
        with pytest.raises(RuntimeError, match="out of range"):
            bh.download(m)
    bh.close()
    h = capi.Handle(prob, 0)
    ib = np.zeros(2, np.int32).ctypes.data_as(C.c_void_p)
    for rc in (L.slu_b200_batch_fill_csr(h.h, prob.n, rpp, cip, vp, pp), L.slu_b200_batch_factor(h.h, ib),
               L.slu_b200_batch_solve(h.h, xp, prob.n, 1), L.slu_b200_batch_download(h.h, 0)):
        assert rc < 0
        assert b"unbatched handle" in L.slu_b200_last_error()
    h.close()
    with pytest.raises(RuntimeError, match="batch = 0"):
        capi.BatchHandle(prob, 0)
    wide, _ = poisson_problem(npdep=2, **kw)
    with pytest.raises(RuntimeError, match="1 x 1 x 1"):
        capi.BatchHandle(wide, 2)
    with pytest.raises(RuntimeError, match="single-GPU"):
        capi.BatchHandle(prob, 2, world_size=2)
