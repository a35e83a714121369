"""The FP64 Schur kernel of the big tiles (schur_kernel_h) on destination layouts the wide-supernode tests do not reach:
tiles whose 64 columns span eight or more destination panels (supernodes of at most 8 columns), and a problem with
many waves of tiles next to supernodes with fewer tiles than SMs; against the oracle, with look-ahead on and off, and
batched.  tc_slices = -1 keeps the int8 path off, so that every big tile (m, n >= 96) takes this kernel."""
import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi, matgen
from util import poisson_problem, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10
# supernodes of at most 8 columns: a 64-column tile spans 8 or more destination panels
_NARROW = dict(N=24, leaf=8, relax=8, maxsup=8)
# 20^3 nodes x 3 dof with 256-column supernodes: about 12,000 128 x 64 tiles in all, next to supernodes with fewer
# tiles than SMs
_MANY = dict(N=20, leaf=32, relax=64, maxsup=256, fem=3)


def _big_tiles(prob):
    """128 x 64 tiles of the updates with m, n >= 96 (host count from the symbolic structure)."""
    ns = np.diff(np.asarray(prob.xsup)).astype(np.int64)
    nsupr = np.asarray(prob.lidx)[np.asarray(prob.lidx_off)[:-1] + 1].astype(np.int64)
    m = nsupr - ns
    n = np.asarray(prob.uval_len, dtype=np.int64) // np.maximum(ns, 1)
    big = (m >= 96) & (n >= 96)
    return ((m[big] + 127) // 128 * ((n[big] + 63) // 64)).astype(np.int64)


@pytest.mark.parametrize("kw", [_NARROW, _MANY], ids=["narrow_destinations", "many_tiles"])
def test_factorization_matches_oracle(kw):
    prob, _ = poisson_problem(**kw)
    chk, _ = poisson_problem(**kw)
    tiles = _big_tiles(prob)
    assert tiles.size > 0, "no update takes the big-tile kernel"
    if kw is _MANY:
        assert tiles.sum() > 8 * 132 and (tiles < 132).any()
    info, st = capi.pdgstrf3d(prob, 0, tc_slices=-1)
    oinfo, oops, _ = oracle.factor(chk)
    assert info == oinfo == 0 and st.reserved[1] == 0
    assert abs(st.ops_fact - oops) <= 1e-9 * oops
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL


@pytest.mark.parametrize("kw", [_NARROW, _MANY], ids=["narrow_destinations", "many_tiles"])
def test_lookahead_on_off_equal(kw):
    on, _ = poisson_problem(**kw)
    off, _ = poisson_problem(**kw)
    assert capi.pdgstrf3d(on, 0, tc_slices=-1)[0] == 0
    assert capi.pdgstrf3d(off, 0, tc_slices=-1, no_lookahead=1)[0] == 0
    a, b = on.layers[0], off.layers[0]
    assert rel_err(a.lval, b.lval) <= 1e-12 and rel_err(a.uval, b.uval) <= 1e-12


def test_batch_of_three_matches_unbatched_narrow():
    """Batched launches (gridDim.y = member) on the narrow destinations."""
    prob, (rp, ci, v) = poisson_problem(**_NARROW)
    vals = matgen.batch_values(rp, ci, v, 3, 1)
    h = capi.BatchHandle(prob, 3)
    h.fill_csr(rp, ci, vals, prob.perm)
    assert not h.factor().any()
    for j in range(3):
        h.download(j)
        got = prob.layers[0].copy()
        ref, _ = poisson_problem(**_NARROW)
        u = capi.Handle(ref, 0, tc_slices=-1)
        u.fill_csr(rp, ci, vals[j], ref.perm)
        assert u.factor() == 0
        u.download()
        u.close()
        assert rel_err(got.lval, ref.layers[0].lval) <= 1e-13 and rel_err(got.uval, ref.layers[0].uval) <= 1e-13, j
    h.close()
