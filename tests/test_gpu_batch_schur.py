"""Partial factorization on batched handles (slu_b200_batch_schur_* and the z twins): every member's S against the dense
Schur complement on the small cases and against the oracle's partial elimination on wide supernodes, the downloaded panels
of every member, the composed solve condense -> S_j -> expand against SciPy, member isolation under independent power-of-
two scalings, a zero pivot and a zero Schur block in single members, a batch of one against an unbatched Schur handle, the
launch and flop counts, the padded host paths, and every refusal.  Each case runs in double and in complex128."""
import ctypes as C
import functools

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from superlu_dist_b200 import capi
from test_gpu_schur import TOL, make, schur_ref, stored_mask
from test_gpu_schur_scale import check_s, first_schur
from test_scaled_parity import exponents, ldexp, mixed_values, permuted, scaled
from test_schur_symbolic_cpu import CASES, oracle_partial, schur_panels, schur_problem

pytestmark = pytest.mark.gpu
DTYPES = ["d", "z"]
CX = {"d": np.float64, "z": np.complex128}


def members(name, dt, B, seed0=7):
    """B members of case `name` (mixed_values seeds seed0 ...) -> (problem, rp, ci, vals (B, nnz), s, [F_j] dense, or
    None outside CASES)"""
    probs = [make(name, CX[dt], seed=seed0 + j, dense=name in CASES) for j in range(B)]
    prob, (rp, ci, _), s, _ = probs[0]
    return prob, rp, ci, np.stack([p[1][2] for p in probs]), s, [p[3] for p in probs]


def factored(prob, rp, ci, vals, s, **opt):
    bh = capi.BatchSchurHandle(prob, len(vals), s, **opt)
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    return bh


def rhs(rng, shape, dt):
    b = rng.standard_normal(shape)
    return b + 1j * rng.standard_normal(shape) if dt == "z" else b


def composed_solve(bh, b):
    """condense, x2 = S_j^-1 g_j per member, expand -> x (B, nrhs, n)"""
    B, nrhs, n = b.shape
    n1 = n - bh.nschur
    S = bh.schur()
    y = bh.condense(b)
    for j in range(B):
        y[j, :, n1:] = np.linalg.solve(S[j], y[j, :, n1:].T).T
    return bh.expand(y)


def sparse_F(prob, rp, ci, vals):
    n = prob.n
    perm = np.asarray(prob.perm)
    rows = np.repeat(np.arange(n), np.diff(rp))
    return sp.csr_matrix((vals, (perm[rows], perm[ci])), shape=(n, n))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_small_cases_against_dense(name, dt):
    B = 3
    prob, rp, ci, vals, s, Fs = members(name, dt, B)
    n1 = prob.n - s
    bh = factored(prob, rp, ci, vals, s)
    S = bh.schur()
    assert S.shape == (B, s, s) and S.dtype == CX[dt]
    off = ~stored_mask(prob, n1)
    for j in range(B):
        Sref = schur_ref(Fs[j], n1)
        scale = np.abs(Sref).max()
        assert np.abs(S[j] - Sref).max() <= TOL * scale, (j, np.abs(S[j] - Sref).max() / scale)
        assert np.all(S[j][off] == 0)
    assert np.abs(S[1] - S[0]).max() > 0.1 * np.abs(S[0]).max()             # the members differ
    bh.close()


@functools.lru_cache(maxsize=None)
def scale_reference(name, dt, B):
    """The oracle's partial elimination of B members of scale case `name` (seeds 7 ...) -> (problem, rp, ci, vals,
    [(S, eliminated L values, eliminated U values)] per member)"""
    prob, (rp, ci, v), _ = schur_problem(name)
    vals = np.stack([mixed_values(rp, ci, v, seed=7 + j, complex_=dt == "z") for j in range(B)])
    k1 = first_schur(prob)
    refs = []
    for j in range(B):
        info, S, lay = oracle_partial(prob, rp, ci, vals[j])
        assert info == 0
        refs.append((S, lay.lval[:lay.lval_off[k1]].copy(), lay.uval[:lay.uval_off[k1]].copy()))
    return prob, rp, ci, vals, refs


SCALE = [pytest.param(name, dt, B, id=f"{name}-{dt}") for name, B in (("p16_w256", 3), ("fem18_w512", 2), ("p32_top", 2))
         for dt in DTYPES if not (name == "fem18_w512" and dt == "z")]


@pytest.mark.parametrize("name,dt,B", SCALE)
def test_scale_cases_against_oracle(name, dt, B):
    """every member's S and downloaded eliminated panels against the oracle run on its own values; the downloaded Schur
    panels bit for bit the member's S"""
    prob, rp, ci, vals, refs = scale_reference(name, dt, B)
    prob.add_layer(0)                                        # a fresh layer for the handle's downloads
    bh = factored(prob, rp, ci, vals, prob.nschur)
    S = bh.schur()
    n1 = prob.n - prob.nschur
    off = ~stored_mask(prob, n1)
    k1 = first_schur(prob)
    lay = prob.layers[0]
    for j, (Sref, lref, uref) in enumerate(refs):
        check_s(S[j], Sref)
        assert np.all(S[j][off] == 0)
        bh.download(j)
        for got, want in ((lay.lval[:lay.lval_off[k1]], lref), (lay.uval[:lay.uval_off[k1]], uref)):
            assert np.abs(got - want).max() <= TOL * np.abs(want).max(), (j, np.abs(got - want).max() / np.abs(want).max())
        assert np.array_equal(schur_panels(prob, lay), S[j])
    bh.close()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", sorted(CASES) + ["p16_w256"])
def test_composed_solve(name, dt):
    """condense -> S_j^-1 -> expand solves every member's whole sparse system: SciPy's spsolve of A_j, residual <= 1e-12"""
    B = 3
    if name in CASES:
        prob, rp, ci, vals, s, _ = members(name, dt, B)
    else:
        prob, rp, ci, vals, _ = scale_reference(name, dt, B)
        prob.add_layer(0)
        s = prob.nschur
    n = prob.n
    perm = np.asarray(prob.perm)
    bh = factored(prob, rp, ci, vals, s)
    rng = np.random.default_rng(3)
    for nrhs in (1, 3):
        b = rhs(rng, (B, nrhs, n), dt)
        x = composed_solve(bh, b)
        for j in range(B):
            F = sparse_F(prob, rp, ci, vals[j])
            fnorm = abs(F).sum(axis=1).max()
            A = sp.csr_matrix((vals[j], ci, rp), shape=(n, n)).tocsc()
            for r in range(nrhs):
                res = np.linalg.norm(F @ x[j, r] - b[j, r]) / (fnorm * np.linalg.norm(x[j, r]) + np.linalg.norm(b[j, r]))
                assert res <= 1e-12, (j, r, res)
                xs = spla.spsolve(A, b[j, r][perm])                   # A_j xs = b in the original ordering
                assert np.abs(x[j, r][perm] - xs).max() <= TOL * np.abs(xs).max(), (j, r)
    st = bh.stats()
    assert st.reserved[4] > 0 and st.reserved[5] > 0
    bh.close()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", ["p8_top", "p20_scat"])
def test_member_isolation_under_scaling(name, dt):
    """member j = 2^er_j A 2^ec_j with independent exponents up to +-20 (member 0: A itself): un-scaled, every S_j is
    S_0; a member reading another member's values or writing another's block of S cannot pass"""
    B = 4
    prob, (rp, ci, v), _ = schur_problem(name)
    if dt == "z":
        prob.dtype = np.dtype(np.complex128)
    prob.add_layer(0)
    n, s = prob.n, prob.nschur
    n1 = n - s
    a = mixed_values(rp, ci, v, seed=9, complex_=dt == "z")
    ex = [(np.zeros(n, np.int64), np.zeros(n, np.int64))] + [exponents(n, 20, seed=j) for j in range(1, B)]
    vals = np.stack([scaled(rp, ci, a, er, ec) for er, ec in ex])
    bh = factored(prob, rp, ci, vals, s)
    S = bh.schur()
    for j in range(1, B):
        er2, ec2 = permuted(prob, ex[j][0])[n1:], permuted(prob, ex[j][1])[n1:]
        assert er2.max() - er2.min() >= 20
        Sj = ldexp(S[j], -(er2[:, None] + ec2[None, :]))
        check_s(Sj, S[0], 1e-12)
        assert np.array_equal(Sj == 0, S[0] == 0)
    bh.close()


@pytest.mark.parametrize("dt", DTYPES)
def test_per_member_zero_pivot_and_zero_schur_block(dt):
    """Member 1 with a zero column in the middle of a 256-column eliminated supernode: its info names the column, the
    others are 0, and the batch_schur_* calls name it.  After a refill the handle works again; a member with
    A21 = A22 = 0 then has S exactly 0 while the others do not."""
    name, B = "p32_top", 3
    prob, rp, ci, vals, refs = scale_reference(name, dt, 2)
    prob.add_layer(0)
    n, s = prob.n, prob.nschur
    n1 = n - s
    xsup = np.asarray(prob.xsup)
    wide = np.nonzero((np.diff(xsup) == 256) & (xsup[:-1] < n1))[0]
    assert len(wide)
    col = int(xsup[wide[0]] + 128)
    perm = np.asarray(prob.perm)
    rows = np.repeat(np.arange(n), np.diff(rp))
    bad = np.where((perm[ci] == col) & (perm[rows] < n1), 0, vals[1]).astype(vals.dtype)
    bh = capi.BatchSchurHandle(prob, B, s)
    bh.fill_csr(rp, ci, np.stack([vals[0], bad, vals[1]]), prob.perm)
    info = bh.factor()
    assert list(info) == [0, col + 1, 0]
    msg = f"member 1 has an exact zero pivot in column {col + 1}"
    with pytest.raises(RuntimeError, match="batch_schur_get: " + msg):
        bh.schur()
    b = np.ones((B, n), CX[dt])
    with pytest.raises(RuntimeError, match="batch_schur_condense: " + msg):
        bh.condense(b)
    with pytest.raises(RuntimeError, match="batch_schur_expand: " + msg):
        bh.expand(b)
    zero_s = np.where(perm[rows] >= n1, 0, vals[1]).astype(vals.dtype)       # A21 = A22 = 0
    bh.fill_csr(rp, ci, np.stack([vals[0], vals[1], zero_s]), prob.perm)
    assert not bh.factor().any()
    S = bh.schur()
    check_s(S[0], refs[0][0])
    check_s(S[1], refs[1][0])
    assert np.all(S[2] == 0)
    assert np.abs(S[0]).max() > 0 and np.abs(S[1]).max() > 0
    bh.close()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", ["p8_top", "p16_w256"])
def test_batch_of_one_matches_unbatched(name, dt):
    prob, rp, ci, vals, s, _ = members(name, dt, 1)
    single = make(name, CX[dt], seed=7, dense=False)[0]
    bh = factored(prob, rp, ci, vals, s)
    h = capi.SchurHandle(single, s)
    h.fill_csr(rp, ci, vals[0], single.perm)
    assert h.factor() == 0
    sb, s1 = bh.stats(), h.stats()
    for f in ("nlevels", "my_supernodes", "ops_fact", "gpu_launches"):
        assert getattr(sb, f) == getattr(s1, f), f
    Sb, S1 = bh.schur(), h.schur()
    assert Sb.shape == (1, s, s)
    assert np.abs(Sb[0] - S1).max() <= TOL * np.abs(S1).max()
    b = rhs(np.random.default_rng(2), (3, prob.n), dt)
    yb, y1 = bh.condense(b[None]), h.condense(b)
    assert np.abs(yb[0] - y1).max() <= TOL * np.abs(y1).max()
    xb, x1 = bh.expand(yb), h.expand(y1)
    assert np.abs(xb[0] - x1).max() <= TOL * np.abs(x1).max()
    assert bh.stats().reserved[5] == h.stats().reserved[5]
    h.close()
    bh.close()


def gather_launches(call):
    """kernel launches of schur_gather_kernel during call(), counted by the CUDA profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    return sum(e.count for e in prof.key_averages() if "schur_gather_kernel" in e.key)


@pytest.mark.parametrize("dt", DTYPES)
def test_counts(dt):
    """ops_fact = B x the unbatched Schur handle's; the factor, condense and expand launches are the unbatched handle's
    whatever B is; the gather is one launch; two schur() calls are bit-identical"""
    name = "p20_scat"
    prob1, (rp, ci, v), _ = schur_problem(name)
    s = prob1.nschur
    if dt == "z":
        prob1.dtype = np.dtype(np.complex128)
    prob1.add_layer(0)
    v0 = mixed_values(rp, ci, v, seed=7, complex_=dt == "z")
    h = capi.SchurHandle(prob1, s)
    h.fill_csr(rp, ci, v0, prob1.perm)
    assert h.factor() == 0
    st1 = h.stats()
    b1 = np.ones(prob1.n, CX[dt])
    h.condense(b1)
    cond1 = h.stats().reserved[5]
    h.expand(b1)
    exp1 = h.stats().reserved[5]
    assert gather_launches(h.schur) == 1
    h.close()
    for B in (1, 3, 17):
        vals = np.stack([mixed_values(rp, ci, v, seed=7 + j, complex_=dt == "z") for j in range(B)])
        bh = factored(prob1, rp, ci, vals, s)
        st = bh.stats()
        assert st.ops_fact == B * st1.ops_fact and st.ops_schur == B * st1.ops_schur, B
        assert st.gpu_launches == st1.gpu_launches and st.nlevels == st1.nlevels, B
        b = np.ones((B, prob1.n), CX[dt])
        bh.condense(b)
        assert bh.stats().reserved[5] == cond1, B
        bh.expand(b)
        assert bh.stats().reserved[5] == exp1, B
        out = {}
        assert gather_launches(lambda: out.setdefault("S", bh.schur())) == 1, B
        S2 = bh.schur()
        assert out["S"].tobytes() == S2.tobytes(), B                          # bit-identical
        st = bh.stats()
        assert st.reserved[6] > 0 and st.reserved[7] > 0
        bh.close()


def _sentinel(dt):
    return np.array(-7.25 + 3.5j if dt == "z" else -7.25, CX[dt])


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", ["p8_top", "p16_w256"])
def test_padded_host_arrays(name, dt):
    """lds = s + 3 and ldx = n + 5 through raw ctypes: the blocks of every member are those of lds = s / ldx = n, the
    padding keeps its sentinels"""
    B = 3
    prob, rp, ci, vals, s, _ = members(name, dt, B)
    n = prob.n
    bh = factored(prob, rp, ci, vals, s)
    L = capi.lib()
    pre = "slu_b200_z_" if dt == "z" else "slu_b200_"
    S = bh.schur()
    buf = np.empty((B, s, s), CX[dt])                   # schur(out=...) writes into the caller's buffer
    assert np.array_equal(bh.schur(out=buf), S) and np.array_equal(buf[1].T, S[1])
    with pytest.raises(ValueError, match="out must be"):
        bh.schur(out=np.empty((B, s, s + 1), CX[dt]))
    lds = s + 3
    out = np.full((B, s, lds), _sentinel(dt))        # member j: column-major s x s with leading dimension lds
    assert getattr(L, pre + "batch_schur_get")(bh.h, out.ctypes.data_as(C.c_void_p), lds) == 0
    for j in range(B):
        assert np.array_equal(out[j, :, :s].T, S[j])
    assert np.all(out[:, :, s:] == _sentinel(dt))
    nrhs, ldx = 3, n + 5
    b = rhs(np.random.default_rng(5), (B, nrhs, n), dt)
    for f, x0 in (("condense", b), ("expand", bh.condense(b))):
        want = getattr(bh, f)(x0)
        buf = np.full((B, nrhs, ldx), _sentinel(dt))
        buf[:, :, :n] = x0
        assert getattr(L, pre + "batch_schur_" + f)(bh.h, buf.ctypes.data_as(C.c_void_p), ldx, nrhs) == 0
        # the update scatter accumulates with atomics, whose order is not fixed: equal up to the last bits
        assert np.abs(buf[:, :, :n] - want).max() <= 1e-14 * np.abs(want).max(), f
        assert np.all(buf[:, :, n:] == _sentinel(dt)), f
    bh.close()


@pytest.mark.parametrize("dt", DTYPES)
def test_refusals(dt):
    L = capi.lib()
    z = dt == "z"
    pre = "slu_b200_z_" if z else "slu_b200_"
    fn = lambda name: getattr(L, pre + name)  # noqa: E731
    err = lambda: L.slu_b200_last_error()  # noqa: E731
    B = 3
    prob, rp, ci, vals, s, _ = members("p8_top", dt, B)
    n = prob.n
    # creation
    for bad in (0, 65536):
        with pytest.raises(RuntimeError, match=f"batch_schur_create: batch = {bad}"):
            capi.BatchSchurHandle(prob, bad, s)
    for bad in (0, n):
        with pytest.raises(RuntimeError, match=f"batch_schur_create: nschur = {bad}"):
            capi.BatchSchurHandle(prob, B, bad)
    k = 1 + int(np.argmax(np.diff(np.asarray(prob.xsup)) > 1))         # a supernode of more than one column
    with pytest.raises(RuntimeError, match=f"batch_schur_create: column .* not a supernode boundary: supernode {k - 1}"):
        capi.BatchSchurHandle(prob, B, n - int(prob.xsup[k - 1]) - 1)
    if not z:
        with pytest.raises(RuntimeError, match="batch_schur_create: the int8"):
            capi.BatchSchurHandle(prob, B, s, tc_slices=7)
    view, keep = capi.make_view(prob, 0)
    opt = capi.make_options(prob)
    hp = C.c_void_p()
    view.nprow = 2
    assert fn("batch_schur_create")(C.byref(hp), C.byref(view), C.byref(opt), B, s) < 0
    assert b"batch_schur_create: batched handles need a 1 x 1 x 1 grid" in err()
    view.nprow = 1
    opt.world_size = 2
    assert fn("batch_schur_create")(C.byref(hp), C.byref(view), C.byref(opt), B, s) < 0
    assert b"batch_schur_create: batched handles are single-GPU" in err()
    del keep
    # before batch_factor
    bh = capi.BatchSchurHandle(prob, B, s)
    with pytest.raises(RuntimeError, match="batch_schur_get needs a .*batch_factor"):
        bh.schur()
    bh.fill_csr(rp, ci, vals, prob.perm)
    with pytest.raises(RuntimeError, match="batch_schur_condense needs a .*batch_factor"):
        bh.condense(np.ones((B, n)))
    assert not bh.factor().any()
    S0 = bh.schur()
    b = np.ones((B, n), CX[dt])
    y0 = bh.condense(b)
    # the batch calls that need complete factors: "Schur handle", and the handle stays usable
    calls = [lambda: bh.solve(b), lambda: bh.solve(b, trans="T"), lambda: bh.rcond(1.0), lambda: bh.selinv(),
             lambda: bh.inv_diag(), lambda: bh.logdet()]
    for call in calls:
        with pytest.raises(RuntimeError, match="on a Schur handle .*batch_schur_"):
            call()
    # the unbatched calls, the schur_* ones included: "batched handle"
    x = np.ones(B * n * s, CX[dt])                                      # large enough for every call below
    xp = x.ctypes.data_as(C.c_void_p)
    assert fn("schur_get")(bh.h, xp, s) < 0 and b"batched handle" in err()
    for f in ("schur_condense", "schur_expand", "solve"):
        assert fn(f)(bh.h, xp, n, 1) < 0 and b"batched handle" in err(), f
    info = C.c_int()
    assert fn("factor")(bh.h, C.byref(info)) < 0 and b"batched handle" in err()
    assert fn("batch_schur_get")(bh.h, xp, s - 1) < 0 and b"lds" in err()
    assert fn("batch_schur_condense")(bh.h, xp, n - 1, 1) < 0
    assert np.array_equal(bh.schur(), S0)
    assert np.abs(bh.condense(b) - y0).max() <= 1e-14 * np.abs(y0).max()
    # the batch_schur_* calls on an ordinary, a plain batched and an unbatched Schur handle
    plain = make("p8_top", CX[dt])[0]
    ho = capi.Handle(plain, 0)
    ho.fill_csr(rp, ci, vals[0], plain.perm)
    assert ho.factor() == 0
    hb = capi.BatchHandle(plain, B)
    hb.fill_csr(rp, ci, vals, plain.perm)
    assert not hb.factor().any()
    hs = capi.SchurHandle(make("p8_top", CX[dt])[0], s)
    hs.fill_csr(rp, ci, vals[0], prob.perm)
    assert hs.factor() == 0
    for hh, want in ((ho, b"on an unbatched handle"), (hb, b"needs a batched Schur handle"), (hs, b"on an unbatched handle")):
        assert fn("batch_schur_get")(hh.h, xp, s) < 0 and want in err()
        for f in ("batch_schur_condense", "batch_schur_expand"):
            assert fn(f)(hh.h, xp, n, 1) < 0 and want in err(), f
    # the existing messages of the unbatched calls
    assert fn("schur_get")(hb.h, xp, s) < 0 and b"needs a Schur handle" in err()
    for hh in (ho, hb, hs):
        hh.close()
    # a member with a zero pivot is named by every new call, and a refill brings the handle back
    perm = np.asarray(prob.perm)
    vz = vals.copy()
    vz[2, perm[ci] == 0] = 0.0
    bh.fill_csr(rp, ci, vz, prob.perm)
    assert list(bh.factor()) == [0, 0, 1]
    with pytest.raises(RuntimeError, match="batch_schur_get: member 2 has an exact zero pivot in column 1"):
        bh.schur()
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    assert np.abs(bh.schur() - S0).max() <= 1e-13 * np.abs(S0).max()
    bh.close()
