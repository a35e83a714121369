"""The panel TRSM on consistent right-hand sides on the GPU (test_trsm_consistent_cpu.py shows the reference meeting every
bound here, and the product with an explicit 16 x 16 inverse failing it): capi.k_trsm (diag_inv_kernel + trsm_kernel)
on every consistent input, then planted factors and indefinite shifts through every factorization route.  A route
passes when its factors meet the factorization bound and come within 16 x max(the oracle's ratio, 8 u) of it, which a
kernel 100 x worse than the oracle but under the loose bound fails, and when its solves N / T / H meet the bound."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

import backward as bw
from oracle import oracle
from superlu_dist_b200 import capi
from test_trsm_consistent_cpu import l_case, planted_problem, u_case
from util import poisson_problem

pytestmark = pytest.mark.gpu
NRHS = [1, 17]
SHIFTS = {"shift_gap": None, "shift_283_64": 283 / 64}


# --------------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("delta", bw.DELTAS)
@pytest.mark.parametrize("z", [False, True], ids=["d", "z"])
@pytest.mark.parametrize("case", ["L", "U"])
def test_k_trsm_consistent(case, z, delta):
    bad = []
    for ns in (bw.ZCWIDTHS if z else bw.CWIDTHS):
        if case == "L":
            u, b = l_case(ns, delta, z)
            r = bw.trsm_l_ratio(u, b, capi.k_trsm(u, b, ucase=False))
        else:
            lo, b = u_case(ns, delta, z)
            r = bw.trsm_u_ratio(lo, b, capi.k_trsm(lo, b, ucase=True))
        bound = bw.kernel_bound(ns, b.dtype)
        if not r <= bound:
            bad.append((ns, r / bound))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ factorizations
def make(name, seed=0, delta=bw.PLANTED_DELTA, mult=bw.PLANTED_MULT):
    """-> (prob with layer 0 holding F, F as CSR, (rowptr, colind, values) of A = P^T F P)"""
    if name in SHIFTS:
        from test_inertia_cpu import shifted
        prob, (rp, ci, v) = poisson_problem(**bw.SHIFT_KW)
        sigma = bw.shift_sigma() if SHIFTS[name] is None else SHIFTS[name]
        vals = shifted(rp, ci, v, sigma)
        prob.fill_layer(0, rp, ci, vals)
        return prob, bw.csr_values(rp, ci, vals, prob.perm, prob.n), (rp, ci, vals)
    prob = planted_problem(name)
    F = bw.plant_factors(prob, delta, mult, seed)
    return prob, F, bw.to_csr(F, prob.perm)


@functools.lru_cache(maxsize=None)
def oracle_ratio(name):
    prob, F, _ = make(name)
    info, _, _ = oracle.factor(prob)
    assert info == 0
    return bw.factor_ratio(F, *bw.factors(prob, prob.layers[0]))[0]


def check(prob, F, base, tiny=0, thresh=None, solve=None):
    """Layer 0 of prob (downloaded) against F: the bound, 16 x max(base, 8 u), then the solves N / T / H"""
    L, U = bw.factors(prob, prob.layers[0])
    r, rep = bw.factor_ratio(F, L, U, thresh)
    bound = bw.factor_bound(prob)
    assert rep == tiny, (rep, tiny)
    assert r <= bound and r <= 16 * max(base, 8 * bw.U), (r / bw.U, base / bw.U, bound / bw.U)
    if solve is not None:
        rng = np.random.default_rng(prob.n)
        for nrhs in NRHS:
            for trans in "NTH":
                b = rng.standard_normal((nrhs, prob.n))
                if np.dtype(prob.dtype).kind == "c":
                    b = b + 1j * rng.standard_normal((nrhs, prob.n))
                rs = bw.solve_ratio(L, U, solve(b, trans), b, trans)
                assert rs <= bound, (nrhs, trans, rs / bw.U, bound / bw.U)


ALL = list(bw.PLANTED) + list(bw.ZPLANTED) + list(SHIFTS)


@pytest.mark.parametrize("depth", [0, 1], ids=["default_depth", "depth1"])
@pytest.mark.parametrize("lookahead", [True, False], ids=["lookahead", "no_lookahead"])
@pytest.mark.parametrize("name", ALL)
def test_pgstrf3d(name, lookahead, depth):
    prob, F, _ = make(name)
    fn = capi.pzgstrf3d if name in bw.ZPLANTED else capi.pdgstrf3d
    info, st = fn(prob, 0, tc_slices=-1, no_lookahead=0 if lookahead else 1, schur_depth=depth)
    assert info == 0
    check(prob, F, oracle_ratio(name), st.tiny_pivots)


@pytest.mark.parametrize("device", [False, True], ids=["factor", "factor_device"])
@pytest.mark.parametrize("name", ALL)
def test_handle_fill_csr(name, device):
    prob, F, (rp, ci, vals) = make(name)
    h = capi.Handle(prob, 0, tc_slices=-1)
    try:
        h.fill_csr(rp, ci, vals, prob.perm)
        if device:
            assert int(h.factor_device().cpu()[0]) == 0
        else:
            assert h.factor() == 0
        h.download()
        check(prob, F, oracle_ratio(name), h.stats().tiny_pivots, solve=h.solve)
    finally:
        h.close()


@pytest.mark.parametrize("name", list(bw.PLANTED) + list(bw.ZPLANTED))
def test_batch_members(name):
    """B = 3 on one pattern: the planted factors, the same without small pivots, another planting"""
    cases = [make(name), make(name, 1, 1.0, 1.0), make(name, 2)]
    prob = cases[0][0]
    assert all(np.array_equal(c[2][1], cases[0][2][1]) for c in cases)
    base = [oracle_ratio(name), None, None]
    for j in (1, 2):
        p2 = cases[j][0]
        assert oracle.factor(p2)[0] == 0
        base[j] = bw.factor_ratio(cases[j][1], *bw.factors(p2, p2.layers[0]))[0]
    rp, ci = cases[0][2][:2]
    h = capi.BatchHandle(prob, 3, tc_slices=-1)
    try:
        h.fill_csr(rp, ci, np.stack([c[2][2] for c in cases]), prob.perm)
        assert not h.factor().any()
        rng = np.random.default_rng(3)
        z = name in bw.ZPLANTED
        for nrhs in NRHS:
            for trans in "NTH":
                b = rng.standard_normal((3, nrhs, prob.n)) + (1j * rng.standard_normal((3, nrhs, prob.n)) if z else 0)
                x = h.solve(b, trans)
                for j in range(3):
                    h.download(j)
                    L, U = bw.factors(prob, prob.layers[0])
                    assert bw.solve_ratio(L, U, x[j], b[j], trans) <= bw.factor_bound(prob), (j, nrhs, trans)
        for j in range(3):
            h.download(j)
            check(prob, cases[j][1], base[j])
    finally:
        h.close()


def test_schur_handle():
    """Planted pivots in the eliminated part of the 256-column top separator of Poisson 16^3 (S = its last 256)"""
    from test_gpu_schur import make as schur_make
    prob, _, s, _ = schur_make("p16_w256", np.float64, dense=False)
    n1 = prob.n - s
    xsup = np.asarray(prob.xsup)
    elim = [k for k in range(prob.nsupers) if xsup[k + 1] <= n1]
    widths = np.diff(xsup)[elim]
    nodes = sorted(np.asarray(elim)[np.argsort(-widths, kind="stable")[:bw.PLANTED_NODES]].tolist())
    F = bw.plant_factors(prob, nodes=nodes)
    rp, ci, vals = bw.to_csr(F, prob.perm)
    # the oracle's partial elimination: the eliminated supernodes in order, S left in the trailing panels
    ref = prob.layers[0].copy()
    info, _, _ = oracle.factor_nodes(prob, ref, np.asarray(elim, np.int32))
    assert info == 0

    def with_s(L, U, S):
        Sc = sp.coo_matrix(S)
        return (U + sp.csr_matrix((Sc.data, (Sc.row + n1, Sc.col + n1)), shape=U.shape)).tocsr()

    Lr, Ur = bw.factors(prob, ref, n_elim=n1)
    Sr = bw.panel_matrix(prob, ref).toarray()[n1:, n1:]
    base = bw.factor_ratio(F, Lr, with_s(Lr, Ur, Sr))[0]
    h = capi.SchurHandle(prob, s, tc_slices=-1)
    try:
        h.fill_csr(rp, ci, vals, prob.perm)
        assert h.factor() == 0
        h.download()
        S = h.schur()
    finally:
        h.close()
    L, U = bw.factors(prob, prob.layers[0], n_elim=n1)
    r, _ = bw.factor_ratio(F, L, with_s(L, U, S))
    assert r <= bw.factor_bound(prob) and r <= 16 * max(base, 8 * bw.U), (r / bw.U, base / bw.U)


REPLACE_DELTA, REPLACE_THRESH = 1e-10, 1e-8


def test_fill_csr_scaled_replaced_pivots_mid_block():
    """replace_tiny_pivot on planted pivots of 1e-10 under a threshold of 1e-8, at in-block offsets 1, 7 and 14"""
    prob, F, (rp, ci, vals) = make("fem6", 0, REPLACE_DELTA)
    prob.replace_tiny_pivot, prob.thresh = 1, REPLACE_THRESH
    ref = prob.layers[0].copy()
    _, _, otiny = oracle.factor(prob, {0: ref})
    assert otiny > 0
    Lr, Ur = bw.factors(prob, ref)
    base = bw.factor_ratio(F, Lr, Ur, REPLACE_THRESH)[0]
    h = capi.Handle(prob, 0)
    try:
        h.fill_csr_scaled(rp, ci, vals, prob.perm, equil=False)
        assert h.factor() == 0
        h.download()
        tiny = h.stats().tiny_pivots
        assert tiny > 0
        d = np.abs(bw.factors(prob, prob.layers[0])[1].diagonal())
        xsup = np.asarray(prob.xsup)
        off = (np.arange(prob.n) - xsup[np.searchsorted(xsup, np.arange(prob.n), side="right") - 1]) % 16
        assert set(off[d == REPLACE_THRESH]) & {1, 7, 14}
        check(prob, F, base, tiny, REPLACE_THRESH, solve=h.solve)
    finally:
        h.close()
