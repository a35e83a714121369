"""Deferred Schur updates along supernode chains (options.reserved[6] = D panels per GEMM, DESIGN 4a) against the oracle at
D = 1..4: chains whose segment lengths are not multiples of BK = 16 (maxsup 100, relax 37), look-ahead on and off, a batch
of three against unbatched, a partial factorization whose Schur block sits above a deferred chain, factor_host with its
overlapped download, and the segmented K loop itself at odd leading dimensions (slu_b200_k_gemm_sub variant 35).  The int8
path is off (tc_slices = -1): deferral is planned on the FP64 route only."""
import os

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import LUProblem, capi, hostlib, matgen
from util import poisson_problem, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10
DEPTHS = [1, 2, 3, 4]
_CHAIN = dict(N=20, leaf=8, relax=37, maxsup=100)             # a 400-column separator in 100-column links
_FEM = dict(N=12, leaf=8, relax=37, maxsup=100, fem=3)         # fem3 separators of 432 columns


@pytest.fixture(autouse=True)
def _no_env(monkeypatch):
    monkeypatch.delenv("SLU_B200_SCHUR_DEPTH", raising=False)


@pytest.mark.parametrize("m,n,k", [(257, 131, 137), (201, 97, 256), (129, 300, 100), (385, 190, 47)])
def test_segmented_k_loop(m, n, k):
    """C -= A B with K cut into three segments of lengths not multiples of 16 (variant 35): the first read in place
    (lda = m, odd), the others repacked with leading dimensions m + 3 and m + 5 and their own ldb."""
    rng = np.random.default_rng(m + n + k)
    a, b, c = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((m, n))
    os.environ["SLU_B200_GEMM_VARIANT"] = "35"
    try:
        out, _ = capi.k_gemm_sub(a, b, c, reps=2)   # the timed repetitions relaunch the same segments
    finally:
        os.environ.pop("SLU_B200_GEMM_VARIANT", None)
    ref = c - a @ b
    assert np.abs(out - ref).max() <= 1e-14 * k * max(np.abs(ref).max(), 1)


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("kw", [_CHAIN, _FEM], ids=["poisson", "fem3"])
def test_factorization_matches_oracle(kw, depth):
    prob, _ = poisson_problem(**kw)
    chk, _ = poisson_problem(**kw)
    deferred = capi.schur_merge(prob, schur_depth=depth)[0]
    assert (deferred > 0) == (depth > 1)
    info, st = capi.pdgstrf3d(prob, 0, tc_slices=-1, schur_depth=depth)
    oinfo, oops, _ = oracle.factor(chk)
    assert info == oinfo == 0 and st.reserved[1] == 0
    assert abs(st.ops_fact - oops) <= 1e-9 * oops
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL


@pytest.mark.parametrize("depth", [2, 4])
def test_lookahead_on_off_and_depth_one_equal(depth):
    """Deferred chains with and without look-ahead equal the undeferred factors up to summation order."""
    ref, _ = poisson_problem(**_FEM)
    assert capi.pdgstrf3d(ref, 0, tc_slices=-1, schur_depth=1)[0] == 0
    for la in (0, 1):
        p, _ = poisson_problem(**_FEM)
        assert capi.pdgstrf3d(p, 0, tc_slices=-1, schur_depth=depth, no_lookahead=la)[0] == 0
        assert rel_err(p.layers[0].lval, ref.layers[0].lval) <= 1e-12 and rel_err(p.layers[0].uval, ref.layers[0].uval) <= 1e-12, la


@pytest.mark.parametrize("depth", [2, 3])
def test_batch_of_three_matches_unbatched(depth):
    prob, (rp, ci, v) = poisson_problem(**_CHAIN)
    vals = matgen.batch_values(rp, ci, v, 3, 1)
    h = capi.BatchHandle(prob, 3, schur_depth=depth)
    h.fill_csr(rp, ci, vals, prob.perm)
    assert not h.factor().any()
    for j in range(3):
        h.download(j)
        got = prob.layers[0].copy()
        ref, _ = poisson_problem(**_CHAIN)
        u = capi.Handle(ref, 0, tc_slices=-1, schur_depth=depth)
        u.fill_csr(rp, ci, vals[j], ref.perm)
        assert u.factor() == 0
        u.download()
        u.close()
        assert rel_err(got.lval, ref.layers[0].lval) <= 1e-13 and rel_err(got.uval, ref.layers[0].uval) <= 1e-13, j
    h.close()


@pytest.mark.parametrize("depth", [2, 4])
def test_factor_host_overlapped_download(depth):
    prob, _ = poisson_problem(**_FEM)
    chk, _ = poisson_problem(**_FEM)
    info, _ = capi.pdgstrf3d(prob, 0, tc_slices=-1, schur_depth=depth, pipeline=1)
    oinfo, _, _ = oracle.factor(chk)
    assert info == oinfo == 0
    assert rel_err(prob.layers[0].lval, chk.layers[0].lval) < TOL and rel_err(prob.layers[0].uval, chk.layers[0].uval) < TOL


def test_partial_factorization_above_chain():
    """The last 100-column link of the top separator is the Schur block: the links below it defer among themselves (not
    into the Schur supernode), and S and the eliminated panels equal those of depth 1."""
    N, ms = 20, 100
    rp, ci, v = hostlib.poisson3d(N)
    perm = hostlib.nd_order(N, leaf=8)

    def make():
        return LUProblem.from_matrix(rp, ci, v, perm, relax=37, maxsup=ms, nschur=ms)

    out = {}
    for depth in (1, 4):
        prob = make()
        if depth > 1:
            assert capi.schur_merge(prob, schur_depth=depth)[0] > 0
        h = capi.SchurHandle(prob, ms, schur_depth=depth)
        h.fill_csr(rp, ci, v, prob.perm)
        assert h.factor() == 0
        S = h.schur()
        h.download()
        h.close()
        out[depth] = (S, prob.layers[0].lval.copy(), prob.layers[0].uval.copy())
    for x, y in zip(out[4], out[1]):
        assert rel_err(x, y) <= 1e-12
