"""slu_b200_batch_selinv, _batch_selinv_get and _batch_logdet (and their slu_b200_z_ twins) on batched handles: every
member's H_j = F_j^-T against a dense inverse and against oracle/selinv.py run on that member's downloaded factors, a
PEXSI-like family of complex shifts, member isolation under independent power-of-two scalings, a batch of one against an
unbatched handle, the launch and flop counts, determinism, untouched factors, and every refusal.  Each case runs in double
and in complex128."""
import ctypes as C

import numpy as np
import pytest

from oracle import selinv
from superlu_dist_b200 import capi
from test_gpu_selinv import csr_of, stored_positions
from test_scaled_parity import exponents, ldexp, make_problem, mixed_values, scaled
from test_selinv_complex_cpu import complex_logdet
from test_unsym_skyline_cpu import make as skyline_make, pattern as skyline_pattern, values as skyline_values
from util import poisson_problem

pytestmark = pytest.mark.gpu
TOL = 1e-10
DTYPES = pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])


def generated(kw, B, complex_, seed0=0):
    """B members with the pattern of poisson_problem(**kw), mixed_values seeds seed0 .. seed0 + B - 1
    -> (prob holding member 0, rp, ci, perm, vals (B, nnz))"""
    _, (rp, ci, v) = poisson_problem(**kw)
    vals = np.stack([mixed_values(rp, ci, v, seed=seed0 + j, complex_=complex_) for j in range(B)])
    prob = make_problem(kw, vals[0])
    return prob, rp, ci, np.asarray(prob.perm, np.int32), vals


def skyline(name, B, complex_):
    rp, ci, _, perm = skyline_pattern(name)
    vals = np.stack([skyline_values(name, complex_, seed=j) for j in range(B)])
    return skyline_make(name, vals[0]), rp, ci, np.asarray(perm, np.int32), vals


def factored(case):
    prob, rp, ci, perm, vals = case
    bh = capi.BatchHandle(prob, len(vals))
    bh.fill_csr(rp, ci, vals, perm)
    assert not bh.factor().any()
    return bh


def batch_h(bh, prob, rows, cols):
    """H_j(rows, cols) of every member through inv_entries with the identity permutation -> (batch, len(rows))"""
    rp, ci, order = csr_of(cols, rows, prob.n)
    vals = bh.inv_entries(rp, ci, np.arange(prob.n, dtype=np.int32))
    assert vals.shape == (bh.batch, len(rows)) and vals.dtype == (np.complex128 if bh.z_ else np.float64)
    out = np.empty_like(vals)
    out[:, order] = vals
    return out


def check_h(got, ref, rows, cols):
    scale = np.abs(ref).max()
    assert np.abs(got - ref).max() <= TOL * scale, np.abs(got - ref).max() / scale
    dg = rows == cols
    assert np.all(np.abs(got[dg] - ref[dg]) <= TOL * np.abs(ref[dg]))


def check_sign(got, want):
    if isinstance(want, complex) or np.iscomplexobj(want):
        assert abs(abs(got) - 1.0) <= 1e-14 and abs(got - want) <= 1e-12, (got, want)
    else:
        assert got == want, (got, want)


SMALL = [pytest.param(lambda c: generated(dict(N=8, leaf=4, relax=8, maxsup=32), 3, c), id="poisson8"),
         pytest.param(lambda c: generated(dict(N=5, leaf=4, relax=8, maxsup=200, fem=3), 3, c), id="fem5"),
         pytest.param(lambda c: skyline("upwind_small", 3, c), id="upwind_small")]


@pytest.mark.parametrize("make", SMALL)
@DTYPES
def test_members_against_dense_inverse(make, complex_):
    case = make(complex_)
    prob = case[0]
    bh = factored(case)
    out = bh.selinv()
    lay = prob.layers[0]
    assert out[0] > 0 and out[1] > 0 and out[3] >= 3 * (16 if complex_ else 8) * (len(lay.lval) - 1)
    rows, cols, _ = stored_positions(prob, lay)
    H = batch_h(bh, prob, rows, cols)
    sign, logabs = bh.logdet()
    assert sign.shape == logabs.shape == (3,) and sign.dtype == (np.complex128 if complex_ else np.float64)
    for j in range(3):
        bh.download(j)
        L, U = prob.dense(lay, True)
        G = np.linalg.inv(L @ U)
        check_h(H[j], G.T[rows, cols], rows, cols)
        s2, l2 = np.linalg.slogdet(L @ U)
        check_sign(sign[j], s2)
        assert abs(logabs[j] - l2) <= 1e-12 * max(1.0, abs(l2))
    bh.close()


def test_pexsi_like_complex_shifts():
    """Members A - z_l I of a real Poisson matrix for three shifts off the real axis (complex symmetric, not Hermitian):
    inv_entries on the pattern of A with A's own permutation against the dense inverses, A^-1(i, j) = H(perm[j], perm[i])
    with a plain transpose, and the logdets against numpy.linalg.slogdet."""
    kw = dict(N=8, leaf=4, relax=8, maxsup=32)
    _, (rp, ci, v) = poisson_problem(**kw)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    shifts = [1.5 + 0.5j, 4.0 + 1.0j, 7.5 - 0.25j]
    vals = np.stack([np.asarray(v, np.complex128) - np.where(rows == ci, z, 0.0) for z in shifts])
    prob = make_problem(kw, vals[0])
    perm = np.asarray(prob.perm, np.int32)
    bh = factored((prob, rp, ci, perm, vals))
    bh.selinv()
    g = bh.inv_entries(rp, ci, perm)
    sign, logabs = bh.logdet()
    for j, z in enumerate(shifts):
        A = np.zeros((n, n), np.complex128)
        A[rows, ci] = vals[j]
        Ainv = np.linalg.inv(A)
        ref = Ainv[rows, ci]
        assert np.abs(g[j] - ref).max() <= TOL * np.abs(ref).max()
        assert np.abs(g[j] - Ainv.T[rows, ci]).max() <= TOL * np.abs(ref).max()           # complex symmetric
        assert np.abs(g[j] - Ainv.conj().T[rows, ci]).max() > 1e-3 * np.abs(ref).max()    # not Hermitian
        s2, l2 = np.linalg.slogdet(A)
        check_sign(sign[j], s2)
        assert abs(logabs[j] - l2) <= 1e-12 * abs(l2)
    bh.close()


BIG = [dict(N=16, leaf=16, relax=32, maxsup=256), dict(N=16, leaf=16, relax=32, maxsup=256, fem=3)]


@pytest.mark.parametrize("kw", BIG, ids=["p16_w256", "fem16"])
@DTYPES
def test_members_against_oracle_on_gpu_factors(kw, complex_):
    case = generated(kw, 4, complex_)
    prob = case[0]
    if not kw.get("fem"):
        assert np.diff(np.asarray(prob.xsup)).max() == 256
    bh = factored(case)
    bh.selinv()
    lay = prob.layers[0]
    rows, cols, u = stored_positions(prob, lay)
    H = batch_h(bh, prob, rows, cols)
    sign, logabs = bh.logdet()
    for j in range(4):
        bh.download(j)
        hl, hu = selinv.selinv(prob, lay)
        check_h(H[j], np.concatenate([hl, hu[u]]), rows, cols)
        s2, l2 = complex_logdet(prob, lay) if complex_ else selinv.logdet(prob, lay)
        check_sign(sign[j], s2)
        assert abs(logabs[j] - l2) <= 1e-12 * abs(l2)
    bh.close()


@pytest.mark.parametrize("E", [10, 20])
@DTYPES
def test_member_isolation_under_scaling(E, complex_):
    """Member j = 2^er_j A 2^ec_j with independent exponents per member (member 0: A itself).  Scaled back, every member's
    A_j^-1 on the pattern of A equals member 0's, and log |det A_j| = log |det A| + (sum er_j + sum ec_j) ln 2: a member
    reading another member's factors, inverse or partials cannot pass."""
    B = 4
    kw = dict(N=10, leaf=8, relax=16, maxsup=128)
    _, (rp, ci, v) = poisson_problem(**kw)
    n = len(rp) - 1
    a = mixed_values(rp, ci, v, seed=9, complex_=complex_)
    ex = [(np.zeros(n, np.int64), np.zeros(n, np.int64))] + [exponents(n, E, seed=j) for j in range(1, B)]
    vals = np.stack([scaled(rp, ci, a, er, ec) for er, ec in ex])
    prob = make_problem(kw, vals[0])
    perm = np.asarray(prob.perm, np.int32)
    bh = factored((prob, rp, ci, perm, vals))
    bh.selinv()
    rows = np.repeat(np.arange(n), np.diff(rp))
    g = bh.inv_entries(rp, ci, perm)                     # A_j^-1(rows, ci) = 2^-ec_j[rows] A^-1(rows, ci) 2^-er_j[ci]
    sign, logabs = bh.logdet()
    g0 = g[0]
    dg = rows == np.asarray(ci)
    for j in range(1, B):
        er, ec = ex[j]
        gj = ldexp(g[j], ec[rows] + er[np.asarray(ci)])
        assert np.abs(gj - g0).max() <= TOL * np.abs(g0).max()
        assert np.all(np.abs(gj[dg] - g0[dg]) <= TOL * np.abs(g0[dg]))
        shift = (er.sum() + ec.sum()) * np.log(2.0)
        assert abs(logabs[j] - (logabs[0] + shift)) <= 1e-12 * abs(logabs[0] + shift)
        if complex_:
            assert abs(sign[j] - sign[0]) <= 1e-12
        else:
            assert sign[j] == sign[0]
    bh.close()


@DTYPES
def test_batch_of_one_matches_unbatched(complex_):
    kw = dict(N=10, leaf=8, relax=16, maxsup=128)
    case = generated(kw, 1, complex_, seed0=4)
    prob, rp, ci, perm, vals = case
    bh = factored(case)
    h = capi.Handle(make_problem(kw, vals[0]), 0)
    h.fill_csr(rp, ci, vals[0], perm)
    assert h.factor() == 0
    ob, o1 = bh.selinv(), h.selinv()
    assert ob[2] == o1[2] and ob[1] == o1[1] and ob[3] == o1[3]
    gb, g1 = bh.inv_entries(rp, ci, perm), h.inv_entries(rp, ci, perm)
    assert gb.shape == (1, len(ci))
    assert np.abs(gb[0] - g1).max() <= TOL * np.abs(g1).max()
    db, d1 = bh.inv_diag(perm), h.inv_diag(perm)
    assert db.shape == (1, prob.n) and np.all(np.abs(db[0] - d1) <= TOL * np.abs(d1))
    (sb, lb), (s1, l1) = bh.logdet(), h.logdet()
    check_sign(sb[0], s1)
    assert abs(lb[0] - l1) <= TOL * abs(l1)
    h.close()
    bh.close()


@DTYPES
def test_launches_flops_determinism(complex_):
    kw = dict(N=10, leaf=8, relax=16, maxsup=128)
    one = generated(kw, 1, complex_)
    h = capi.Handle(make_problem(kw, one[4][0]), 0)
    h.fill_csr(one[1], one[2], one[4][0], one[3])
    assert h.factor() == 0
    flops1 = h.selinv()[1]
    nlevels = h.stats().nlevels
    h.close()
    for B in (1, 3, 17):
        case = generated(kw, B, complex_)
        prob, rp, ci, perm, vals = case
        bh = factored(case)
        lay = prob.layers[0]
        before = []
        for j in (0, B - 1):
            bh.download(j)
            before.append((lay.lval.copy(), lay.uval.copy()))
        rng = np.random.default_rng(6)
        b = rng.standard_normal((B, prob.n))
        if complex_:
            b = b + 1j * rng.standard_normal(b.shape)
        x0 = bh.solve(b)
        out = bh.selinv()
        assert out[2] == 7 * nlevels - 1 and out[1] == B * flops1, (B, out, nlevels, flops1)
        g = bh.inv_entries(rp, ci, perm)
        assert np.isfinite(g).all()
        assert bh.selinv()[2] == out[2]
        assert np.array_equal(g, bh.inv_entries(rp, ci, perm))      # bit-identical
        for j, (l0, u0) in zip((0, B - 1), before):
            bh.download(j)
            assert np.array_equal(lay.lval, l0) and np.array_equal(lay.uval, u0)
        x1 = bh.solve(b)
        # the solve accumulates with atomics, whose order is not fixed: equal up to the last bits
        assert np.abs(x1 - x0).max() <= 1e-14 * np.abs(x0).max()
        bh.close()


@DTYPES
def test_refusals(complex_):
    L = capi.lib()
    z = "z_" if complex_ else ""
    fn = lambda name: getattr(L, f"slu_b200_{z}{name}")  # noqa: E731
    err = lambda: L.slu_b200_last_error()  # noqa: E731
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    prob, rp, ci, perm, vals = generated(kw, 3, complex_)
    n, nd = prob.n, 2 if complex_ else 1
    out = (C.c_double * 4)()
    ident = np.arange(n, dtype=np.int32)
    la, sg = (C.c_double * 3)(), (C.c_double * 6)()
    # unbatched handle
    h = capi.Handle(make_problem(kw, vals[0]), 0)
    h.fill_csr(rp, ci, vals[0], perm)
    assert h.factor() == 0
    assert fn("batch_selinv")(h.h, out) < 0 and b"unbatched handle" in err()
    assert fn("batch_logdet")(h.h, la, sg) < 0 and b"unbatched handle" in err()
    ip = ident.ctypes.data_as(C.c_void_p)
    rp1 = np.arange(n + 1, dtype=np.int32)
    assert fn("batch_selinv_get")(h.h, n, rp1.ctypes.data_as(C.c_void_p), ip, ip, (C.c_double * (nd * n))()) < 0
    assert b"unbatched handle" in err()
    h.close()
    # before batch_factor
    bh = capi.BatchHandle(prob, 3)
    with pytest.raises(RuntimeError, match="batch_selinv needs a .*batch_factor"):
        bh.selinv()
    bh.fill_csr(rp, ci, vals, perm)
    with pytest.raises(RuntimeError, match="batch_selinv needs a .*batch_factor"):
        bh.selinv()
    with pytest.raises(RuntimeError, match="batch_logdet needs a .*batch_factor"):
        bh.logdet()
    assert not bh.factor().any()
    # _get before batch_selinv, and after a later batch_fill_csr / batch_factor
    with pytest.raises(RuntimeError, match="batch_selinv on the current factors"):
        bh.inv_diag()
    bh.selinv()
    assert bh.inv_diag().shape == (3, n) and np.isfinite(bh.inv_diag()).all()
    assert fn("batch_selinv_get")(bh.h, n - 1, rp1.ctypes.data_as(C.c_void_p), ip, ip, (C.c_double * (3 * nd * n))()) < 0
    assert b"does not match" in err()
    # an entry with no slot: counted once, not once per member
    rows, cols, _ = stored_positions(prob, prob.layers[0])
    have = set(zip(rows.tolist(), cols.tolist()))
    r, c = next((r, c) for r in range(n) for c in range(n) if (r, c) not in have)
    with pytest.raises(RuntimeError, match=r"batch_selinv_get: 1 entries have no slot"):
        bh.inv_entries(np.array([0] * (c + 1) + [1] * (n - c), np.int32), np.array([r], np.int32), ident)
    assert not bh.factor().any()
    with pytest.raises(RuntimeError, match="batch_selinv on the current factors"):
        bh.inv_diag()
    bh.selinv()
    bh.fill_csr(rp, ci, vals, perm)                  # new values: the members wait for their batch_factor
    with pytest.raises(RuntimeError, match="batch_selinv_get needs a .*batch_factor"):
        bh.inv_diag()
    assert not bh.factor().any()
    with pytest.raises(RuntimeError, match="batch_selinv on the current factors"):
        bh.inv_diag()
    # member 1 with an exact zero pivot: column 0 of F_1 = P A_1 P^T is zero
    vz = vals.copy()
    vz[1, perm[ci] == 0] = 0.0
    bh.fill_csr(rp, ci, vz, perm)
    info = bh.factor()
    assert info[0] == 0 and info[1] == 1 and info[2] == 0
    with pytest.raises(RuntimeError, match="batch_selinv: member 1 has an exact zero pivot"):
        bh.selinv()
    with pytest.raises(RuntimeError, match="batch_logdet: member 1 has an exact zero pivot"):
        bh.logdet()
    bh.close()
