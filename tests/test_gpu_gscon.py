"""slu_b200_gscon and its doublecomplex / batched twins: the dlacn2 / zlacn2 condition estimate on the resident factors,
checked against the NumPy restatement of tests/test_gscon_cpu.py (itself checked against LAPACK's gecon) driven by
SciPy solves with F = P A P^T assembled from the same CSR."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from superlu_dist_b200 import capi
from test_gpu_solve_complex import CASES as ZCASES, complex_csr
from test_gpu_solve_trans import CASES, permuted, real_case
from test_gscon_cpu import lacn2
from util import complex_problem, load_fixture, poisson_problem

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DENSE_MAX = 5000     # orders up to which the exact ||F^-1|| comes from a dense inverse


def anorm_of(F, norm):
    return float(np.asarray(abs(sp.csr_matrix(F)).sum(axis=0 if norm == "1" else 1)).max())


def restated(F, norm):
    """(est, kases) of the restatement for F (sparse or dense), solving with SciPy's splu: kases is the sequence of its
    solves, "1" for kase 1 and "2" for kase 2 (so len(kases) is the solve count)"""
    F = sp.csc_matrix(F)
    cplx = np.iscomplexobj(F.data)
    lu = spl.splu(F)
    kases = []
    ops = [lambda v: lu.solve(v), lambda v: lu.solve(v, trans="H" if cplx else "T")]
    if norm != "1":
        ops.reverse()
    k1 = lambda v: (kases.append("1"), ops[0](v))[1]            # noqa: E731
    k2 = lambda v: (kases.append("2"), ops[1](v))[1]            # noqa: E731
    est, ns = lacn2(k1, k2, F.shape[0], cplx)
    assert ns == len(kases)
    return est, "".join(kases)


def lockstep(seqs):
    """The batched schedule for the members' kase sequences: each round solves one kase, the members whose next kase it
    is take it; the next round takes the other kase if any member waits for it, else the same one.
    -> (rounds, whether some member had to wait through a round of the other kase)"""
    pos, kase, rounds, waited = [0] * len(seqs), "1", 0, False
    while True:
        rounds += 1
        for m, s in enumerate(seqs):
            if pos[m] < len(s):
                if s[pos[m]] == kase:
                    pos[m] += 1
                else:
                    waited = True
        pending = {s[p] for s, p in zip(seqs, pos) if p < len(s)}
        if not pending:
            return rounds, waited
        other = "2" if kase == "1" else "1"
        kase = other if other in pending else kase


def check_estimate(h, F, norm):
    """rcond of the handle against the restatement (1e-10), its solve count, and est <= the exact norm"""
    anorm = anorm_of(F, norm)
    rc = h.rcond(anorm, norm)
    est_ref, kases = restated(F, norm)
    ns = len(kases)
    rc_ref = (1.0 / est_ref) / anorm
    assert abs(rc - rc_ref) <= 1e-10 * rc_ref, (norm, rc, rc_ref)
    assert h.stats().reserved[7] == ns, (norm, h.stats().reserved[7], ns)
    assert h.stats().reserved[6] > 0
    if F.shape[0] <= DENSE_MAX:
        exact = np.abs(np.linalg.inv(sp.csr_matrix(F).toarray())).sum(axis=0 if norm == "1" else 1).max()
        assert 1.0 / (rc * anorm) <= exact * (1 + 1e-12), (norm, 1.0 / (rc * anorm), exact)
    return rc


@pytest.mark.parametrize("kw", CASES)
def test_rcond_double(kw):
    prob, rp, ci, vals, F = real_case(kw)
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    rc1 = check_estimate(h, F, "1")
    check_estimate(h, F, "I")
    assert abs(h.rcond(anorm_of(F, "1"), "O") - rc1) <= 1e-13 * rc1     # 'O' is '1'
    h.close()


def test_rcond_unsymmetric_pattern():
    prob, _, post = load_fixture("unsym360_mmd")
    assert int(post["info"][0]) == 0
    every = np.ones(prob.nsupers, bool)
    F = prob.matvec([(prob.layers[0], every)], np.eye(prob.n), 0).T
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    for norm in ("1", "I"):
        check_estimate(h, F, norm)
    h.close()


@pytest.mark.parametrize("kw", ZCASES)
def test_rcond_complex(kw):
    prob = complex_problem(**kw)
    rp, ci, v = complex_csr(**kw)
    F = permuted(rp, ci, v, prob.perm)
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    for norm in ("1", "I"):
        check_estimate(h, F, norm)
    h.close()


def test_near_singular_sweep():
    """Members A - sigma_k I of a symmetric Poisson A with sigma_k = lambda_min (1 - delta_k): nonsingular M-matrices,
    whose inverses are entrywise nonnegative, so dlacn2 finds the exact 1-norm; rcond falls with delta_k."""
    kw = dict(N=10, leaf=8, relax=16, maxsup=64)
    prob, (rp, ci, v) = poisson_problem(**kw)
    n = prob.n
    A = sp.csr_matrix((v, ci, rp), shape=(n, n))
    lmin = float(spl.eigsh(A, k=1, sigma=0, which="LM", return_eigenvectors=False)[0])
    deltas = 10.0 ** -np.arange(1, 7)
    diag = np.repeat(np.arange(n), np.diff(rp)) == ci
    vals = np.stack([v - diag * lmin * (1 - d) for d in deltas])
    bh = capi.BatchHandle(prob, len(deltas))
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    anorm = np.array([anorm_of(sp.csr_matrix((vk, ci, rp), shape=(n, n)), "1") for vk in vals])
    rc = bh.rcond(anorm, "1")
    for k, vk in enumerate(vals):
        exact = np.abs(np.linalg.inv(permuted(rp, ci, vk, prob.perm).toarray())).sum(axis=0).max()
        est = 1.0 / (rc[k] * anorm[k])
        assert abs(est - exact) <= 1e-6 * exact, (k, est, exact)
    assert np.all(np.diff(rc) < 0), rc
    bh.close()


def mixed_values(rp, ci, seed, cplx):
    """Random off-diagonal values of both signs (complex: random phases) on the pattern; the diagonal is 0.6 ... 1 times
    the row's off-diagonal 1-norm, plus 0.5.  dlacn2 takes 5, 7 or 9 solves on such matrices, depending on the seed,
    alternating 1, 2, 1, 2, ... and ending at its test on the index of the largest entry."""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    off = rows != np.asarray(ci)
    rng = np.random.default_rng(seed)
    w = rng.standard_normal(len(ci)) + (1j * rng.standard_normal(len(ci)) if cplx else 0)
    w = np.where(off, w, 0)
    return np.where(off, w, np.bincount(rows, np.abs(w), len(rp) - 1)[rows] * rng.uniform(0.6, 1.0, len(rp) - 1)[rows] + 0.5)


def stopping_values(rp, ci, v, cplx):
    """A member on which the estimator stops at its test after the first e_j solve, so that its solves run 1, 2, 1, 1:
    real, the Poisson values themselves (an M-matrix: the sign vector repeats); complex, the diagonal 2, 2i, -2, -2i, ...
    with zero off-diagonal entries, whose inverse has columns of equal 1-norm, so that the estimate does not grow (zlacn2
    has no repeated-sign test, and for n a power of 2 every value on the way is exact)."""
    if not cplx:
        return np.asarray(v, np.float64)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    return np.where(rows == np.asarray(ci), np.array([2.0, 2.0j, -2.0, -2.0j])[rows % 4], 0.0)


LKW = dict(N=8, leaf=4, relax=8, maxsup=32)                # n = 512
LOCKSTEP_SEEDS = {False: [0, 1, 3, 7], True: [0, 2, 4]}    # restated solve counts differ between these members


@pytest.mark.parametrize("cplx", [False, True])
def test_batched_lockstep_matches_unbatched(cplx):
    """Members whose kase sequences differ, one of them not alternating: that member has to keep its pending vector
    through a round of the other kase.  The rounds must be those of the lock-step schedule of the restated sequences."""
    prob, (rp, ci, v) = poisson_problem(**LKW)
    one = (lambda: complex_problem(**LKW)) if cplx else (lambda: poisson_problem(**LKW)[0])
    vals = np.stack([mixed_values(rp, ci, s, cplx) for s in LOCKSTEP_SEEDS[cplx]] + [stopping_values(rp, ci, v, cplx)])
    B = len(vals)
    bh = capi.BatchHandle(one(), B)
    bh.fill_csr(rp, ci, vals, prob.perm)
    assert not bh.factor().any()
    for norm in ("1", "I"):
        Fs = [permuted(rp, ci, vk, prob.perm) for vk in vals]
        anorm = np.array([anorm_of(F, norm) for F in Fs])
        ref = [restated(F, norm) for F in Fs]
        seqs = [kases for _, kases in ref]
        assert seqs[-1] == "1211", seqs
        assert len({len(s) for s in seqs}) > 1, seqs
        want_rounds, waited = lockstep(seqs)
        assert waited, seqs
        rc = bh.rcond(anorm, norm)
        rounds = bh.stats().reserved[7]
        assert rounds == want_rounds, (norm, rounds, want_rounds, seqs)
        assert max(map(len, seqs)) <= rounds <= 2 * max(map(len, seqs))
        for j in range(B):
            h = capi.Handle(one(), 0)
            h.fill_csr(rp, ci, vals[j], prob.perm)
            assert h.factor() == 0
            rc1 = h.rcond(anorm[j], norm)
            assert h.stats().reserved[7] == len(seqs[j])
            h.close()
            assert abs(rc[j] - rc1) <= 1e-12 * rc1, (norm, j, rc[j], rc1)
            assert abs(rc[j] * anorm[j] * ref[j][0] - 1) <= 1e-10
    bh.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_solve_and_factors_unaffected(cplx):
    """gscon reads the factors only: L and U are bit for bit those of before, the solves agree with those of before
    (bit for bit where the solve itself reproduces bit for bit; its atomic adds have no fixed order), and
    stats.reserved[4] / [5] still describe the last solve."""
    kw = CASES[1]
    prob = complex_problem(**kw) if cplx else real_case(kw)[0]
    rng = np.random.default_rng(5)
    b = rng.standard_normal(prob.n) + (1j * rng.standard_normal(prob.n) if cplx else 0)
    h = capi.Handle(prob, 0)
    h.upload()
    assert h.factor() == 0
    trans = "H" if cplx else "T"
    x0 = {t: h.solve(b, trans=t) for t in ("N", trans)}
    x1 = {t: h.solve(b, trans=t) for t in ("N", trans)}
    st = h.stats()
    h.download()
    lay = prob.layers[0]
    l0, u0 = lay.lval.copy(), lay.uval.copy()
    for norm in ("1", "I"):
        assert h.rcond(1.0, norm) > 0
    st2 = h.stats()
    assert (st2.reserved[4], st2.reserved[5]) == (st.reserved[4], st.reserved[5])
    h.download()
    assert np.array_equal(lay.lval, l0) and np.array_equal(lay.uval, u0)
    for t in ("N", trans):
        x2 = h.solve(b, trans=t)
        if np.array_equal(x0[t], x1[t]):
            assert np.array_equal(x2, x0[t]), t
        else:
            assert np.abs(x2 - x0[t]).max() <= 1e-14 * np.abs(x0[t]).max(), t
    h.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_errors(cplx):
    kw = dict(N=6, leaf=4, relax=4, maxsup=8)
    prob = complex_problem(**kw) if cplx else poisson_problem(**kw)[0]
    L = capi.lib()
    pre = "slu_b200_z_" if cplx else "slu_b200_"
    gscon, batch_gscon = getattr(L, pre + "gscon"), getattr(L, pre + "batch_gscon")
    out = C.c_double(-1.0)
    two = np.ones(2)
    h = capi.Handle(prob, 0)
    with pytest.raises(RuntimeError, match="needs a successful"):
        h.rcond(1.0)                                            # not factored yet
    h.upload()
    assert h.factor() == 0
    for bad in (b"2", b"X", b"F"):
        assert gscon(h.h, bad, 1.0, C.byref(out)) < 0
        assert b"norm must be" in L.slu_b200_last_error()
    with pytest.raises(ValueError):
        h.rcond(1.0, norm="one")
    for a in (-1.0, float("nan")):
        with pytest.raises(RuntimeError, match="anorm"):
            h.rcond(a)
    for a in (0.0, float("inf")):
        assert h.rcond(a) == 0.0
        assert h.stats().reserved[7] == 0                       # no solve
    assert h.rcond(1.0, "i") > 0
    assert batch_gscon(h.h, b"1", two.ctypes.data_as(C.c_void_p), two.ctypes.data_as(C.c_void_p)) < 0
    assert b"unbatched handle" in L.slu_b200_last_error()
    h.close()
    bh = capi.BatchHandle(prob, 2)
    with pytest.raises(RuntimeError, match="batch_factor"):
        bh.rcond(1.0)                                           # not factored yet
    assert gscon(bh.h, b"1", 1.0, C.byref(out)) < 0
    assert b"batched handle" in L.slu_b200_last_error()
    rp, ci, v = complex_csr(**kw) if cplx else poisson_problem(**kw)[1]
    bh.fill_csr(rp, ci, np.stack([v, v]), prob.perm)
    assert not bh.factor().any()
    with pytest.raises(RuntimeError, match=r"anorm\[1\]"):
        bh.rcond([1.0, -2.0])
    rc = bh.rcond([0.0, 1.0])
    assert rc[0] == 0.0 and rc[1] > 0
    bh.close()


@pytest.mark.parametrize("cplx", [False, True])
def test_batched_refuses_zero_pivot_member(cplx):
    kw = dict(N=12, leaf=8, relax=16, maxsup=128)
    prob, (rp, ci, v) = poisson_problem(**kw)
    if cplx:
        prob, (rp, ci, v) = complex_problem(**kw), complex_csr(**kw)
    vals = np.stack([v, v, v])
    vals[1][np.asarray(prob.perm)[ci] == 0] = 0.0              # column 1 of P A_1 P^T is zero: exact zero pivot there
    bh = capi.BatchHandle(prob, 3)
    bh.fill_csr(rp, ci, vals, prob.perm)
    info = bh.factor()
    assert info[1] == 1 and not np.delete(info, 1).any(), info
    with pytest.raises(RuntimeError, match="member 1"):
        bh.rcond(1.0)
    bh.close()


@pytest.mark.parametrize("world", [2, 4])
def test_rcond_1x1xPz(world):
    """The Z-distributed estimate, double and doublecomplex, against the single-process result."""
    if capi.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29940 + world), os.path.join(HERE, "mgpu_gscon_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert out.stdout.count("rcond err") == world
