"""Child process of tests/test_gpu_variants_complex.py: the doublecomplex kernels and pzgstrf3d_b200 against NumPy, the
oracle and the reference's own factors, the pzdrive3d drop-in, and the overlapped upload.  Runs in its own process so
that a fault in a kernel cannot poison the CUDA context of the suite."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def z_kernel_cases():
    """doublecomplex kernels (slu_kernels_z.cu) against NumPy/SciPy, through slu_b200_z_k_*."""
    import scipy.linalg as sl
    from superlu_dist_b200 import capi

    def crand(rng, *shape):
        return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)

    def lu_nopivot(a):
        a = a.copy()
        n = a.shape[1]
        for j in range(n - 1):
            if a[j, j] != 0:
                a[j + 1:n, j] /= a[j, j]
            a[j + 1:n, j + 1:] -= np.outer(a[j + 1:n, j], a[j, j + 1:])
        return a

    for ns, extra in [(1, 0), (5, 3), (16, 0), (17, 40), (33, 7), (100, 1), (256, 19)]:
        rng = np.random.default_rng(ns)
        a = crand(rng, ns + extra, ns)
        a[:ns] += ns * np.eye(ns)
        ref = a.copy()
        ref[:ns] = lu_nopivot(a[:ns])
        out, info, tiny = capi.k_diag_lu(a)
        assert info == 0 and tiny == 0
        assert np.abs(out - ref).max() <= 1e-12 * ns * np.abs(ref).max(), ("diag_lu", ns, extra)
    a = crand(np.random.default_rng(3), 8, 8) + 8 * np.eye(8)
    a[:, 0] = 0.0
    out, info, tiny = capi.k_diag_lu(a.copy(), col0=100)
    assert info == 101
    for ns, m in [(1, 1), (7, 3), (16, 64), (31, 65), (64, 200), (256, 130)]:
        rng = np.random.default_rng(ns * 1000 + m)
        lu = crand(rng, ns, ns) + ns * np.eye(ns)
        x = crand(rng, m, ns)
        ref = sl.solve_triangular(np.triu(lu), x.T, trans="T", lower=False).T
        out = capi.k_trsm(lu, x, ucase=False)
        assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1), ("trsm_l", ns, m)
        lu = crand(rng, ns, ns) / ns + np.eye(ns)
        x = crand(rng, ns, m)
        ref = sl.solve_triangular(np.tril(lu, -1) + np.eye(ns), x, lower=True, unit_diagonal=True)
        out = capi.k_trsm(lu, x, ucase=True)
        assert np.abs(out - ref).max() <= 1e-12 * ns * max(np.abs(ref).max(), 1), ("trsm_u", ns, m)
    for (m, n, k) in [(1, 1, 1), (7, 5, 3), (33, 31, 17), (96, 96, 16), (128, 32, 8), (130, 257, 100), (300, 200, 256),
                      (95, 400, 30), (513, 129, 33)]:
        rng = np.random.default_rng(m * 7 + n * 3 + k)
        a, b, c = crand(rng, m, k), crand(rng, k, n), crand(rng, m, n)
        out, _ = capi.k_gemm_sub(a, b, c)
        ref = c - a @ b
        assert np.abs(out - ref).max() <= 1e-13 * k * max(np.abs(ref).max(), 1), ("zgemm_sub", m, n, k)
    print("doublecomplex kernels ok")


def z_factor_cases():
    """pzgstrf3d_b200 against the reference's own factors (cg20 through pzdrive3d) and the complex oracle."""
    from oracle import oracle
    from superlu_dist_b200 import capi
    from util import FIXTURES, complex_problem, load_fixture, rel_err
    for name in [f for f in FIXTURES if f.startswith("cg")]:
        prob, ref, post = load_fixture(name)
        info, st = capi.pzgstrf3d(prob, 0)
        lay = prob.layers[0]
        err = max(rel_err(lay.lval, ref.lval), rel_err(lay.uval, ref.uval))
        assert info == int(post["info"][0]) and err < 1e-10, (name, info, err)
        assert abs(st.ops_fact - float(post["ops_fact"][0])) <= 2e-5 * float(post["ops_fact"][0]), name
    for kw in (dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=12, leaf=8, relax=16, maxsup=128),
               dict(N=5, leaf=4, relax=8, maxsup=200, fem=3)):
        prob, chk = complex_problem(**kw), complex_problem(**kw)
        h = capi.Handle(prob, 0)
        h.upload()
        info = h.factor()
        h.download()
        st = h.stats()
        h.close()
        oinfo, oops, _ = oracle.factor(chk)
        a, b = prob.layers[0], chk.layers[0]
        err = max(rel_err(a.lval, b.lval), rel_err(a.uval, b.uval))
        assert info == oinfo == 0 and err < 1e-10, (kw, info, oinfo, err)
        assert abs(st.ops_fact - oops) <= 1e-9 * oops, (st.ops_fact, oops)
    print("pzgstrf3d_b200 ok")


def z_dropin_case():
    """The unmodified pzdrive3d on libslu_b200.so (hook compiled with -DSLU_HOOK_COMPLEX binds pzgstrf3d_b200)."""
    import tempfile
    from test_dropin import ZDRV, run_driver
    if not os.path.exists(ZDRV):
        print("oracle/_ref/pzdrive3d not built; skipped")
        return
    with tempfile.TemporaryDirectory() as tmp:
        for grid in ((20, 20, 1), (12, 12, 12)):
            err, log = run_driver(tmp, "b200", grid, complex_=True)
            assert "pzgstrf3d_b200:" in log and err < 1e-11, (grid, err)
    print("pzdrive3d drop-in ok")


def overlap_h2d_cases():
    """slu_b200_factor_host with options.reserved[3]: zeroed arena, staged atomic-add upload per level, factorization
    and download all overlapped -- against the oracle, and against the plain path on the same matrix."""
    from oracle import oracle
    from superlu_dist_b200 import capi
    from util import poisson_problem, rel_err
    for kw in (dict(N=12, leaf=8, relax=8, maxsup=32), dict(N=16, leaf=8, relax=16, maxsup=256),
               dict(N=6, leaf=4, relax=8, maxsup=200, fem=3)):
        prob, _ = poisson_problem(**kw)
        chk, _ = poisson_problem(**kw)
        h = capi.Handle(prob, 0, overlap_h2d=1)
        info = h.factor_host()
        st = h.stats()
        # a second factorization on the same handle (arena re-zeroed, host arrays restored)
        again, _ = poisson_problem(**kw)
        prob.layers[0].lval[:] = again.layers[0].lval
        prob.layers[0].uval[:] = again.layers[0].uval
        info2 = h.factor_host()
        h.close()
        oinfo, oops, _ = oracle.factor(chk)
        a, b = prob.layers[0], chk.layers[0]
        err = max(rel_err(a.lval, b.lval), rel_err(a.uval, b.uval))
        assert info == info2 == oinfo == 0 and err < 1e-10, (kw, info, info2, oinfo, err)
        assert abs(st.ops_fact - oops) <= 1e-9 * oops
    print("overlapped upload ok")


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("zkernels", "all"):
        z_kernel_cases()
    if what in ("zfactor", "all"):
        z_factor_cases()
    if what in ("zdropin", "all"):
        z_dropin_case()
    if what in ("h2d", "all"):
        overlap_h2d_cases()
