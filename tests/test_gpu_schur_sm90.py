"""The FP64 Schur kernel of the big tiles on mma.sync.m16n8k8.f64 (schur_kernel_h, gemm_tile_h): the GEMM main loop
against NumPy at edge shapes, and whole factorizations with 256- and 512-column supernodes against the oracle, with and
without look-ahead and batched.  The int8 path is off by default; tc_slices = -1 turns it off explicitly, so that every
big tile takes this kernel whatever the default."""
import os

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi, matgen
from util import poisson_problem, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10
_W256 = dict(N=16, leaf=16, relax=32, maxsup=256)         # a 256-column top separator
_W512 = dict(N=18, leaf=32, relax=64, maxsup=512, fem=3)  # supernodes of 486 and 512 columns


@pytest.mark.parametrize("variant", [0, 30])
@pytest.mark.parametrize("m,n,k", [(128, 64, 128), (257, 131, 137), (200, 97, 256), (129, 300, 512), (385, 190, 16)])
def test_gemm_sub_m16n8k8(variant, m, n, k):
    """C -= A B through the Hopper main loop (variant 0 takes it for m, n >= 96): tiles cut by M and N, K not a multiple
    of BK = 16, odd lda (= m)."""
    rng = np.random.default_rng(m * 7 + n * 3 + k)
    a, b, c = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((m, n))
    os.environ["SLU_B200_GEMM_VARIANT"] = str(variant)
    try:
        out, _ = capi.k_gemm_sub(a, b, c)
    finally:
        os.environ.pop("SLU_B200_GEMM_VARIANT", None)
    ref = c - a @ b
    assert np.abs(out - ref).max() <= 1e-14 * k * max(np.abs(ref).max(), 1)


@pytest.mark.parametrize("tc", [0, -1])
@pytest.mark.parametrize("kw", [_W256, _W512])
def test_factorization_matches_oracle(kw, tc):
    """tc = 0: the default routing (FP64: the int8 path is opt-in); -1: this kernel for every big tile, explicitly."""
    prob, _ = poisson_problem(**kw)
    chk, _ = poisson_problem(**kw)
    assert np.diff(np.asarray(prob.xsup)).max() == kw["maxsup"]
    info, st = capi.pdgstrf3d(prob, 0, tc_slices=tc)
    oinfo, oops, _ = oracle.factor(chk)
    assert info == oinfo == 0 and st.reserved[1] == 0
    assert abs(st.ops_fact - oops) <= 1e-9 * oops
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL


@pytest.mark.parametrize("kw", [_W256, _W512])
def test_lookahead_on_off_equal(kw):
    """The urgent / bulk split (modes 1 and 2) covers the same tiles as mode 0: equal factors up to summation order."""
    on, _ = poisson_problem(**kw)
    off, _ = poisson_problem(**kw)
    assert capi.pdgstrf3d(on, 0, tc_slices=-1)[0] == 0
    assert capi.pdgstrf3d(off, 0, tc_slices=-1, no_lookahead=1)[0] == 0
    a, b = on.layers[0], off.layers[0]
    assert rel_err(a.lval, b.lval) <= 1e-12 and rel_err(a.uval, b.uval) <= 1e-12


def test_batch_of_three_matches_unbatched():
    prob, (rp, ci, v) = poisson_problem(**_W256)
    vals = matgen.batch_values(rp, ci, v, 3, 1)
    h = capi.BatchHandle(prob, 3)
    h.fill_csr(rp, ci, vals, prob.perm)
    assert not h.factor().any()
    for j in range(3):
        h.download(j)
        got = prob.layers[0].copy()
        ref, _ = poisson_problem(**_W256)
        u = capi.Handle(ref, 0, tc_slices=-1)
        u.fill_csr(rp, ci, vals[j], ref.perm)
        assert u.factor() == 0
        u.download()
        u.close()
        assert rel_err(got.lval, ref.layers[0].lval) <= 1e-13 and rel_err(got.uval, ref.layers[0].uval) <= 1e-13, j
    h.close()
