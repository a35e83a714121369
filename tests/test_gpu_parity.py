"""Parity of the CUDA pdgstrf3d (through the C-ABI) with (a) factors of the UNMODIFIED reference
(tests/golden) and (b) the oracle on generated matrices, plus size-independent properties at
larger sizes.  Tolerances: entry-wise 1e-10 relative to max|factor| (FP64; only the summation
order differs: DMMA tiles + atomics vs BLAS), residual ||LU-A||_F/||A||_F <= 1e-12."""
import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi
from util import REAL_FIXTURES, load_fixture, poisson_problem, rel_err, residual_probe

pytestmark = pytest.mark.gpu
TOL = 1e-10


@pytest.mark.parametrize("name", REAL_FIXTURES)
def test_matches_reference_factors(name):
    prob, ref, post = load_fixture(name)
    lay = prob.layers[0]
    info, st = capi.pdgstrf3d(prob, 0)
    assert info == int(post["info"][0])
    assert st.tiny_pivots == int(post["TinyPivots"][0])
    ref_ops = float(post["ops_fact"][0])
    assert abs(st.ops_fact - ref_ops) <= (0.02 if name.startswith("unsym") else 2e-5) * ref_ops
    assert rel_err(lay.lval, ref.lval) < TOL
    assert rel_err(lay.uval, ref.uval) < TOL
    assert st.gpu_launches > 0


@pytest.mark.parametrize("N,leaf,relax,maxsup,fem", [(6, 4, 4, 8, None), (10, 8, 8, 32, None), (16, 32, 16, 64, None),
                                                      (18, 16, 32, 256, None), (6, 8, 12, 48, 3), (12, 64, 1, 4, None),
                                                      (12, 8, 8, 32, None), (14, 8, 16, 256, None), (6, 4, 8, 200, 3)])
def test_matches_oracle_on_generated(N, leaf, relax, maxsup, fem):
    prob, _ = poisson_problem(N, leaf, relax, maxsup, fem=fem)
    chk, _ = poisson_problem(N, leaf, relax, maxsup, fem=fem)
    info, st = capi.pdgstrf3d(prob, 0)
    oinfo, oops, _ = oracle.factor(chk)
    assert info == oinfo == 0
    assert abs(st.ops_fact - oops) <= 1e-9 * oops
    assert abs(st.ops_fact - prob.ops_fact) <= 1e-9 * oops
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < TOL and rel_err(a.uval, b.uval) < TOL


def test_handle_api_and_refactor():
    """create / upload / factor / download (dCreateLUgpuHandle ... dCopyLUGPU2Host), twice."""
    prob, mat = poisson_problem(12, 8, 8, 32)
    chk, _ = poisson_problem(12, 8, 8, 32)
    oracle.factor(chk)
    pristine = prob.layers[0].copy()
    h = capi.Handle(prob, 0)
    for _ in range(2):
        prob.layers[0].lval[:] = pristine.lval
        prob.layers[0].uval[:] = pristine.uval
        h.upload()
        assert h.factor() == 0
        h.download()
        assert rel_err(prob.layers[0].lval, chk.layers[0].lval) < TOL
        assert rel_err(prob.layers[0].uval, chk.layers[0].uval) < TOL
    st = h.stats()
    assert st.t_factor_s > 0 and st.gpu_launches > 0 and st.nlevels > 0
    h.close()


def test_factor_host_overlapped_download():
    """slu_b200_factor_host == upload + factor + download (D2H of every level overlapped with the factorization)."""
    prob, _ = poisson_problem(14, 8, 8, 32)
    chk, _ = poisson_problem(14, 8, 8, 32)
    oracle.factor(chk)
    h = capi.Handle(prob, 0)
    assert h.factor_host() == 0
    h.close()
    assert rel_err(prob.layers[0].lval, chk.layers[0].lval) < TOL
    assert rel_err(prob.layers[0].uval, chk.layers[0].uval) < TOL
    # and through the one-call entry point with options.reserved[2]
    prob2, _ = poisson_problem(14, 8, 8, 32)
    info, _ = capi.pdgstrf3d(prob2, 0, pipeline=1)
    assert info == 0
    assert rel_err(prob2.layers[0].lval, chk.layers[0].lval) < TOL


@pytest.mark.parametrize("name", [f for f in REAL_FIXTURES if f.startswith("unsym")] + ["g20_pddrive3d"])
def test_factor_host_on_unsymmetric_pattern(name):
    """pdgstrf3d_b200 with options.reserved[2] (overlapped transfers) on patterns whose U skylines are NOT full:
    the library falls back to upload + factor + download (skyline <-> packed conversion) instead of failing."""
    prob, ref, post = load_fixture(name)
    info, st = capi.pdgstrf3d(prob, 0, pipeline=1)
    assert info == int(post["info"][0])
    assert rel_err(prob.layers[0].lval, ref.lval) < TOL and rel_err(prob.layers[0].uval, ref.uval) < TOL
    # and with the level-by-level arena of the overlapped upload requested too
    prob, ref, post = load_fixture(name)
    info, st = capi.pdgstrf3d(prob, 0, pipeline=1, overlap_h2d=1)
    assert info == int(post["info"][0])
    assert rel_err(prob.layers[0].lval, ref.lval) < TOL and rel_err(prob.layers[0].uval, ref.uval) < TOL


def test_retired_schur_variant_is_refused():
    """options.schur_variant once selected other Schur tile kernels; the field keeps its place in the struct and must be 0."""
    prob, _ = poisson_problem(N=6, leaf=4, relax=8, maxsup=32)
    with pytest.raises(RuntimeError, match="schur_variant is retired and must be 0"):
        capi.Handle(prob, 0, schur_variant=4)


@pytest.mark.parametrize("kw", [dict(N=10, leaf=8, relax=8, maxsup=32), dict(N=16, leaf=16, relax=32, maxsup=256),
                                dict(N=6, leaf=4, relax=8, maxsup=200, fem=3)])
def test_solve_on_resident_factors(kw):
    """slu_b200_solve (the consumer of pdgstrf3d, pdgstrs3d.c:6604): forward/back substitution on the factors that are
    still in HBM.  b = A xtrue in the ordering of the factored matrix; several right-hand sides; twice on one handle."""
    prob, _ = poisson_problem(**kw)
    lay = prob.layers[0]
    every = np.ones(prob.nsupers, bool)
    rng = np.random.default_rng(1)
    xtrue = rng.standard_normal((3, prob.n))
    b = prob.matvec([(lay, every)], xtrue, 0)
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError):
        h.solve(b)                      # not factored yet
    h.upload()
    assert h.factor() == 0
    for rhs in (b, b[0]):
        x = h.solve(rhs)
        ref = xtrue if rhs.ndim == 2 else xtrue[0]
        assert np.abs(x - ref).max() <= 1e-10 * np.abs(ref).max(), np.abs(x - ref).max()
    assert h.stats().reserved[4] > 0
    h.close()


def test_matrix_file_through_the_readers(tmp_path):
    """File -> reader (libslu_b200_host: Matrix Market and Harwell-Boeing) -> symbolic -> pdgstrf3d_b200 -> solve:
    the path a caller with an on-disk matrix takes (the role of dcreate_matrix + dreadMM/dreadhb in EXAMPLE/)."""
    import scipy.io
    import scipy.sparse as sp
    from superlu_dist_b200 import LUProblem, hostlib, matgen
    rp, ci, v = hostlib.poisson3d(9)
    perm = hostlib.nd_order(9, leaf=8)
    a = sp.csr_matrix((v, ci, rp))
    scipy.io.mmwrite(str(tmp_path / "p9.mtx"), a)
    matgen.write_harwell_boeing(str(tmp_path / "p9.rua"), rp, ci, v)
    ref, _ = poisson_problem(9, 8, 8, 32)
    oracle.factor(ref)
    for name in ("p9.mtx", "p9.rua"):
        nr, nc, rp2, ci2, v2 = hostlib.read_matrix(str(tmp_path / name))
        assert nr == nc == 729 and np.array_equal(rp2, rp) and np.array_equal(ci2, ci)
        prob = LUProblem.from_matrix(rp2, ci2, v2, perm, relax=8, maxsup=32)
        info, _ = capi.pdgstrf3d(prob, 0)
        assert info == 0
        assert rel_err(prob.layers[0].lval, ref.layers[0].lval) < TOL and rel_err(prob.layers[0].uval, ref.layers[0].uval) < TOL


@pytest.mark.parametrize("kw", [dict(N=10, leaf=8, relax=8, maxsup=32), dict(N=6, leaf=4, relax=8, maxsup=200, fem=3)])
def test_device_side_distribution(kw):
    """slu_b200_fill_csr (the job of pddistribute3d on the GPU, SURVEY 8f N1) puts exactly the values into HBM that
    uploading the host-distributed panels does: download right after it and compare; then factor from it."""
    prob, (rp, ci, v) = poisson_problem(**kw)
    want = prob.layers[0].copy()
    prob.layers[0].lval[:] = -7.0                     # poison the host arrays: they must not be read
    prob.layers[0].uval[:] = -7.0
    h = capi.Handle(prob, 0)
    h.fill_csr(rp, ci, v, prob.perm)
    h.download()
    assert np.array_equal(prob.layers[0].lval, want.lval) and np.array_equal(prob.layers[0].uval, want.uval)
    assert h.factor() == 0
    h.download()
    h.close()
    chk, _ = poisson_problem(**kw)
    oracle.factor(chk)
    assert rel_err(prob.layers[0].lval, chk.layers[0].lval) < TOL and rel_err(prob.layers[0].uval, chk.layers[0].uval) < TOL


def test_zero_pivot_info():
    prob, _ = poisson_problem(6, 4, 4, 8)
    lay = prob.layers[0]
    # zero the whole first column of the first supernode -> exact zero pivot at global column 1
    ns0 = prob.xsup[1] - prob.xsup[0]
    nsupr0 = prob.lidx[prob.lidx_off[0] + 1]
    lay.lval[lay.lval_off[0]:lay.lval_off[0] + nsupr0] = 0.0
    assert ns0 >= 1
    info, _ = capi.pdgstrf3d(prob, 0)
    assert info == 1


@pytest.mark.parametrize("N", [32, 40])
def test_residual_property_at_scale(N):
    """Size-independent property: ||(LU - A) x|| / ||A x|| for random +-1 probes (estimates
    ||LU-A||_F/||A||_F) and max|U diag| sanity, at sizes where the oracle would take minutes."""
    prob, _ = poisson_problem(N, leaf=64, relax=32, maxsup=256)
    pre = prob.layers[0].copy()
    info, st = capi.pdgstrf3d(prob, 0, verbose=0)
    assert info == 0
    everything = np.ones(prob.nsupers, bool)
    res = residual_probe(prob, [(pre, everything)], [(prob.layers[0], everything)])
    assert res < 1e-12, res
    assert abs(st.ops_fact - prob.ops_fact) <= 1e-9 * prob.ops_fact


def test_degenerate_matrices():
    """Ragged inputs through the CUDA path: diagonal matrix (supernodes without any off-diagonal block, NULL U
    panels), n = 1, and a tridiagonal chain (one etree path, many levels with one tiny supernode each)."""
    import scipy.sparse as sp
    from superlu_dist_b200 import LUProblem
    for A in (sp.diags([np.arange(1.0, 8.0)], [0]).tocsr(), sp.csr_matrix(np.array([[3.0]])),
              sp.diags([-np.ones(29), 4 * np.ones(30), -np.ones(29)], [-1, 0, 1]).tocsr()):
        A.sort_indices()
        rp, ci, v = A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(np.float64)
        for relax, maxsup in ((1, 4), (8, 8)):
            prob = LUProblem.from_matrix(rp, ci, v, None, relax=relax, maxsup=maxsup)
            chk = LUProblem.from_matrix(rp, ci, v, None, relax=relax, maxsup=maxsup)
            info, st = capi.pdgstrf3d(prob, 0)
            oinfo, oops, _ = oracle.factor(chk)
            assert info == oinfo == 0
            assert abs(st.ops_fact - oops) <= 1e-9 * max(oops, 1)
            assert rel_err(prob.layers[0].lval, chk.layers[0].lval) < TOL
            assert rel_err(prob.layers[0].uval, chk.layers[0].uval) < TOL
