"""CPU-side checks of the C-ABI library: it loads, exports every symbol include/slu_b200.h declares,
its struct layouts match the ctypes mirrors, and compute entry points fail loudly without a GPU."""
import numpy as np
import pytest

from superlu_dist_b200 import capi
from util import poisson_problem


def test_library_loads_and_exports_declared_symbols():
    L = capi.lib()
    syms = capi.declared_symbols()
    assert "pdgstrf3d_b200" in syms and len(syms) >= 15
    for s in syms:
        assert hasattr(L, s), s
    assert L.slu_b200_abi_version() == 1


def test_no_cpu_fallback():
    if capi.device_count() > 0:
        pytest.skip("a GPU is visible")
    prob, _ = poisson_problem(4, 4, 4, 8)
    with pytest.raises(RuntimeError):
        capi.pdgstrf3d(prob, 0)
    with pytest.raises(RuntimeError):
        capi.k_gemm_sub(np.ones((2, 2)), np.ones((2, 2)), np.ones((2, 2)))


def test_host_library_exports_declared_symbols():
    """libslu_b200_host.so exports every function include/slu_b200_host.h declares."""
    import ctypes
    import os
    import re
    from superlu_dist_b200._paths import HOST_SO, INCLUDE
    from superlu_dist_b200 import hostlib
    hostlib.lib()
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(INCLUDE, "slu_b200_host.h")).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(sluh_\w+)\s*\(", text)))
    L = ctypes.CDLL(HOST_SO)
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(L, s), s


# ---- slu_b200_plan: the library's analysis (layout, level plan, flop accounting) needs no device ---------------
@pytest.mark.parametrize("kw", [dict(N=10, leaf=8, relax=8, maxsup=32), dict(N=6, leaf=4, relax=8, maxsup=200, fem=3)])
@pytest.mark.parametrize("cplx", [False, True])
def test_plan_matches_oracle_accounting(kw, cplx):
    """ops_fact of the CUDA library's analysis == the oracle's flop count (pinned to the reference's
    stat->ops[FACT] by test_oracle_vs_reference), for pdgstrf3d and for the doublecomplex build; the arena holds
    exactly the L panels plus the dense-packed U panels; the level-by-level layout (overlapped upload) keeps every
    level contiguous (checked inside slu_b200_plan)."""
    from oracle import oracle
    from util import complex_problem
    prob = complex_problem(**kw) if cplx else poisson_problem(**kw)[0]
    chk = complex_problem(**kw) if cplx else poisson_problem(**kw)[0]
    _, oops, _ = oracle.factor(chk)
    for opt in ({}, {"overlap_h2d": 1}):
        st = capi.plan(prob, 0, **opt)
        assert abs(st.ops_fact - oops) <= 1e-12 * oops
        assert st.lu_device_bytes == (st.nnz_l + st.nnz_u) * (16 if cplx else 8)
        assert st.nnz_l == int(prob.lval_len.sum()) and st.my_supernodes == prob.nsupers and st.nlevels >= 1
    with pytest.raises(RuntimeError, match="schur_variant is retired and must be 0"):
        capi.plan(prob, 0, schur_variant=4)


def test_plan_supernode_width_limits():
    """The double path takes supernodes up to MAX_SUPER_SIZE = 512 (superlu_defs.h:154); the doublecomplex build stops at
    256 columns and says so instead of mis-factoring."""
    from oracle import oracle
    from util import complex_problem
    kw = dict(N=14, leaf=32, relax=64, maxsup=512, fem=3)
    prob, chk = poisson_problem(**kw)[0], poisson_problem(**kw)[0]
    assert np.diff(np.asarray(prob.xsup)).max() == 512
    _, oops, _ = oracle.factor(chk)
    st = capi.plan(prob, 0)
    assert abs(st.ops_fact - oops) <= 1e-12 * oops
    zprob = complex_problem(N=18, leaf=32, relax=64, maxsup=512)
    assert np.diff(np.asarray(zprob.xsup)).max() > 256
    with pytest.raises(RuntimeError, match="wider than 256"):
        capi.plan(zprob, 0)


def test_plan_golden_complex_fixture():
    """The reference's own pzgstrf3d flop count on cg20.cua (float32 accumulation there: 2e-5)."""
    from util import FIXTURES, load_fixture
    for name in [f for f in FIXTURES if f.startswith("cg")]:
        prob, _, post = load_fixture(name)
        st = capi.plan(prob, 0)
        ref = float(post["ops_fact"][0])
        assert abs(st.ops_fact - ref) <= 2e-5 * ref, (name, st.ops_fact, ref)


@pytest.mark.parametrize("npdep", [2, 4])
def test_plan_layers_partition_the_work(npdep):
    """1 x 1 x Pz: every supernode is counted by exactly one layer (pdgstrf3d.c:336, reduceStat sums over Z), with
    the reference-style and the cooperative schedule and with the level-by-level layout."""
    kw = dict(N=12, leaf=8, relax=8, maxsup=32)
    whole, _ = poisson_problem(**kw)
    total = capi.plan(whole, 0).ops_fact
    prob, _ = poisson_problem(npdep=npdep, **kw)
    for opt in (dict(world_size=npdep), dict(world_size=npdep, no_coop=1), dict(world_size=npdep, overlap_h2d=1)):
        parts = [capi.plan(prob, z, world_rank=z, **opt) for z in range(npdep)]
        assert abs(sum(p.ops_fact for p in parts) - total) <= 1e-12 * total
        assert sum(p.my_supernodes for p in parts) == prob.nsupers
