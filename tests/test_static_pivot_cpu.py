"""Static pivoting on the host: the maximum-product matching with its scalings (sluh_large_diag_perm, the role of
dldperm_dist job 5 / MC64 in pdgssvx3d) against SciPy's optimal assignment and, where the reference library was built,
against the reference itself; and the NumPy restatement of dgsequ / dlaqgs the device equilibration is checked with."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import maximum_bipartite_matching, min_weight_full_bipartite_matching

from superlu_dist_b200 import hostlib

HERE = os.path.dirname(os.path.abspath(__file__))
EXAMPLES = os.path.join(HERE, "golden", "readers", "example_matrices.npz")
REF_SO = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libsuperlu_ref.so")
EPS = np.finfo(np.float64).eps
SMLNUM = np.finfo(np.float64).tiny           # dmach_dist("S")
BIGNUM = 1.0 / SMLNUM
SMALL = SMLNUM / EPS                         # dlaqgs_dist: dmach("Safe minimum") / dmach("Precision")
LARGE = 1.0 / SMALL


# ---- matrices ------------------------------------------------------------------------------------------------------
def example(name, tmp_path):
    """One of the reference's example matrices (g4.rua, g20.rua, big.rua, cg20.cua) as SciPy CSR"""
    path = str(tmp_path / name)
    with open(path, "wb") as f:
        f.write(np.load(EXAMPLES)[name].tobytes())
    nr, nc, rp, ci, v = hostlib.read_matrix(path)
    return sp.csr_matrix((v, ci, rp), shape=(nr, nc))


def random_unsym(n, seed, density=4.0, spread=20.0):
    """Random unsymmetric values over 2^+-spread on a random pattern that holds a hidden perfect matching"""
    rng = np.random.default_rng(seed)
    A = sp.random(n, n, density=min(1.0, density / n), random_state=seed, format="csr") + sp.eye(n, format="csr")
    A = sp.csr_matrix(A[rng.permutation(n)])
    A.data = rng.standard_normal(A.nnz) * np.exp2(rng.uniform(-spread, spread, A.nnz))
    return A


def permuted_triangular(n, seed):
    rng = np.random.default_rng(seed)
    L = sp.tril(sp.random(n, n, density=min(1.0, 6.0 / n), random_state=seed), -1) + sp.diags(rng.uniform(1e-3, 1.0, n))
    L = sp.csr_matrix(L)
    L.data = L.data * rng.choice([-1.0, 1.0], L.nnz) * np.exp2(rng.uniform(-8, 8, L.nnz))
    return sp.csr_matrix(L[rng.permutation(n)])


def block_matrix(nblk, bs, seed):
    rng = np.random.default_rng(seed)
    A = sp.block_diag([sp.csr_matrix(rng.standard_normal((bs, bs))) for _ in range(nblk)], format="csr")
    A = A + sp.random(nblk * bs, nblk * bs, density=2.0 / (nblk * bs), random_state=seed)
    return sp.csr_matrix(sp.csr_matrix(A)[rng.permutation(nblk * bs)])


def poisson2d(g):
    T = sp.diags([-1.0, 4.0, -1.0], [-1, 0, 1], shape=(g, g))
    S = sp.diags([-1.0, -1.0], [-1, 1], shape=(g, g))
    return sp.csr_matrix(sp.kron(sp.eye(g), T) + sp.kron(S, sp.eye(g)))


def kkt(g, m, seed, sigma=0.0):
    """[K - sigma I, B^T; B, 0]: a Poisson block K, m random constraints B (two entries per row and the row's own unknown,
    full row rank), a zero (2, 2) block -- no unpivoted LU in the natural order"""
    rng = np.random.default_rng(seed)
    n = g * g
    K = poisson2d(g) - sigma * sp.eye(n)
    cols = rng.choice(n, m, replace=False)
    rows = np.concatenate([np.arange(m)] * 3)
    cc = np.concatenate([cols, rng.integers(0, n, m), rng.integers(0, n, m)])
    B = sp.csr_matrix((np.concatenate([np.full(m, 1.0), rng.uniform(-0.5, 0.5, 2 * m)]), (rows, cc)), shape=(m, n))
    B.sum_duplicates()
    return sp.csr_matrix(sp.bmat([[K, B.T], [B, None]], format="csr"))


def csr_parts(A):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data


# ---- the optimum and the restatements ------------------------------------------------------------------------------
def optimal_logprod(A):
    """max over perfect matchings of sum log |a_{i sigma(i)}| by SciPy (weights log colmax - log|a| + 1 > 0)"""
    A = sp.csr_matrix(abs(A))
    A.eliminate_zeros()
    colmax = A.max(axis=0).toarray().ravel()
    W = A.copy()
    W.data = np.log(colmax[W.indices]) - np.log(W.data) + 1.0
    r, c = min_weight_full_bipartite_matching(W)
    return np.log(np.asarray(A[r, c]).ravel()).sum()


def abs1(v):
    v = np.asarray(v)
    return np.abs(v.real) + np.abs(v.imag) if np.iscomplexobj(v) else np.abs(v)


def scale_values(v, rows, cols, R, C):
    """(R[i] a_ij) C[j], componentwise for complex values (the scalings are real)"""
    if np.iscomplexobj(v):
        w = np.ascontiguousarray(v).view(np.float64).reshape(-1, 2)
        return ((w * R[rows, None]) * C[cols, None]).ravel().view(np.complex128)
    return (v * R[rows]) * C[cols]


def equilibrate(rp, ci, v, R, C):
    """NumPy restatement of the device equilibration: dgsequ_dist on M = Pr Dr A Dc (|re| + |im| in complex, as
    slud_z_abs1), dlaqgs_dist's choice, the factors folded into R and C.  -> (R, C, rowcnd, colcnd, amax, equed)"""
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    m = abs1(scale_values(v, rows, ci, R, C))
    r = np.zeros(n)
    np.maximum.at(r, rows, m)
    rcmin, rcmax = min(BIGNUM, r.min()), max(0.0, r.max())
    amax = rcmax
    assert rcmin > 0, "zero row"
    rinv = 1.0 / np.minimum(np.maximum(r, SMLNUM), BIGNUM)
    rowcnd = max(rcmin, SMLNUM) / min(rcmax, BIGNUM)
    c = np.zeros(n)
    np.maximum.at(c, ci, m * rinv[rows])
    ccmin, ccmax = min(BIGNUM, c.min()), max(0.0, c.max())
    assert ccmin > 0, "zero column"
    cinv = 1.0 / np.minimum(np.maximum(c, SMLNUM), BIGNUM)
    colcnd = max(ccmin, SMLNUM) / min(ccmax, BIGNUM)
    if rowcnd >= 0.1 and SMALL <= amax <= LARGE:
        equed = 0 if colcnd >= 0.1 else 2
    else:
        equed = 1 if colcnd >= 0.1 else 3
    return (R * rinv if equed & 1 else R.copy()), (C * cinv if equed & 2 else C.copy()), rowcnd, colcnd, amax, equed


# ---- tests -----------------------------------------------------------------------------------------------------------
def check_matching(A):
    rp, ci, v = csr_parts(A)
    perm_r, R, Cs, lp = hostlib.large_diag_perm(rp, ci, v)
    n = A.shape[0]
    assert np.array_equal(np.sort(perm_r), np.arange(n))
    ref = optimal_logprod(A)
    assert abs(lp - ref) <= 1e-12 * max(1.0, abs(ref)), (lp, ref)
    S = abs(sp.diags(R) @ sp.csr_matrix(abs(A)) @ sp.diags(Cs)).tocsr()
    assert S.max() <= 1.0 + 4 * EPS
    d = np.asarray(S[np.arange(n), perm_r]).ravel()
    assert np.abs(d - 1.0).max() <= 4 * EPS
    again = hostlib.large_diag_perm(rp, ci, v)
    assert all(np.array_equal(a, b) for a, b in zip(again[:3], (perm_r, R, Cs))) and again[3] == lp
    return perm_r, R, Cs


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("n", [7, 60, 400])
def test_random_unsymmetric_is_optimal(n, seed):
    check_matching(random_unsym(n, seed))


@pytest.mark.parametrize("seed", range(3))
def test_structurally_tricky_patterns_are_optimal(seed):
    check_matching(permuted_triangular(300, seed))
    check_matching(block_matrix(40, 7, seed))


@pytest.mark.parametrize("g,m", [(6, 5), (12, 30), (20, 60)])
def test_kkt_is_optimal_and_fills_the_zero_block(g, m):
    A = kkt(g, m, g)
    assert np.count_nonzero(A.diagonal()) == g * g
    perm_r, R, Cs = check_matching(A)
    P = hostlib.row_permute(*csr_parts(A), perm_r)
    F = sp.csr_matrix((P[2], P[1], P[0]), shape=A.shape)
    assert np.count_nonzero(F.diagonal()) == A.shape[0]
    assert (abs(F - sp.csr_matrix(A)[np.argsort(perm_r)]) > 0).nnz == 0


def test_structurally_singular_returns_the_rank():
    A = sp.csr_matrix(kkt(6, 5, 1))
    A = sp.lil_matrix(A)
    A[3, :] = 0                                                    # an empty row
    A[:, 7] = 0                                                    # and an empty column
    A = sp.csr_matrix(A)
    A.eliminate_zeros()
    rank = int((maximum_bipartite_matching(A, perm_type="column") >= 0).sum())
    rp, ci, v = csr_parts(A)
    n = A.shape[0]
    out = np.zeros(2)
    rc = hostlib.lib().sluh_large_diag_perm(n, rp, ci, np.abs(v), np.empty(n, np.int32), np.empty(n), np.empty(n), out)
    assert rc == rank < n and out[0] == -np.inf
    with pytest.raises(ValueError, match=f"structural rank {rank}"):
        hostlib.large_diag_perm(rp, ci, v)


def test_explicit_zeros_are_not_edges():
    A = sp.csr_matrix(np.array([[0.0, 2.0], [3.0, 1.0]]))
    rp, ci, v = np.array([0, 2, 4], np.int32), np.array([0, 1, 0, 1], np.int32), np.array([0.0, 2.0, 3.0, 1.0])
    perm_r, R, Cs, lp = hostlib.large_diag_perm(rp, ci, v)
    assert list(perm_r) == [1, 0] and abs(lp - np.log(6.0)) < 1e-15
    assert abs(optimal_logprod(A) - lp) < 1e-15


def test_row_permute_and_complex_values(tmp_path):
    A = example("cg20.cua", tmp_path)
    rp, ci, v = csr_parts(A)
    perm_r, R, Cs, lp = hostlib.large_diag_perm(rp, ci, v)
    assert abs(lp - optimal_logprod(A)) <= 1e-12 * max(1.0, abs(lp))
    prp, pci, pv = hostlib.row_permute(rp, ci, v, perm_r)
    assert pv.dtype == np.complex128
    F = sp.csr_matrix((pv, pci, prp), shape=A.shape)
    P = sp.csr_matrix((np.ones(len(perm_r)), (perm_r, np.arange(len(perm_r)))), shape=A.shape)
    assert abs(F - P @ A).max() == 0


def test_equilibration_restatement_choices():
    """THRESH and the amax tests pick rows, columns, both or neither"""
    A = sp.csr_matrix(poisson2d(5))
    rp, ci, v = csr_parts(A)
    one = np.ones(25)
    assert equilibrate(rp, ci, v, one, one)[5] == 0
    rs = np.exp2(np.where(np.arange(25) % 2 == 0, 30.0, -30.0))
    assert equilibrate(rp, ci, v, rs, one)[5] in (1, 3)
    assert equilibrate(rp, ci, v, one, rs)[5] == 2
    assert equilibrate(rp, ci, v * 1e-300, one, one)[5] in (1, 3)


# ---- against the reference's own routines ----------------------------------------------------------------------------
class _NC(C.Structure):
    _fields_ = [("nnz", C.c_int32), ("nzval", C.c_void_p), ("rowind", C.c_void_p), ("colptr", C.c_void_p)]


class _SuperMatrix(C.Structure):
    _fields_ = [("Stype", C.c_int), ("Dtype", C.c_int), ("Mtype", C.c_int), ("nrow", C.c_int32), ("ncol", C.c_int32),
                ("Store", C.c_void_p)]


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF_SO):
        pytest.skip("the reference library was not built (oracle/_ref/libsuperlu_ref.so)")
    return C.CDLL(REF_SO)


def ref_ldperm(ref, A):
    """dldperm_dist(5, ...) on A (CSC, 32-bit int_t) -> (perm, exp(u), exp(v) / ... as returned: u, v logs)"""
    Acsc = sp.csc_matrix(A)
    Acsc.sort_indices()
    n = A.shape[0]
    cp = Acsc.indptr.astype(np.int32).copy()
    ri = Acsc.indices.astype(np.int32).copy()
    val = np.abs(Acsc.data).astype(np.float64)
    perm = np.empty(n, np.int32)
    u, v = np.empty(n), np.empty(n)
    ref.dldperm_dist.argtypes = [C.c_int, C.c_int, C.c_int32] + [C.c_void_p] * 6
    rc = ref.dldperm_dist(5, n, len(ri), cp.ctypes.data, ri.ctypes.data, val.ctypes.data, perm.ctypes.data, u.ctypes.data,
                          v.ctypes.data)
    assert rc == 0
    return perm, u, v


@pytest.mark.parametrize("name", ["g4.rua", "g20.rua", "big.rua"])
def test_same_objective_as_the_reference(ref, tmp_path, name):
    A = example(name, tmp_path)
    rp, ci, v = csr_parts(A)
    perm_r, R, Cs, lp = hostlib.large_diag_perm(rp, ci, v)
    perm, u, vv = ref_ldperm(ref, A)
    absA = sp.csr_matrix(abs(A))
    ref_lp = np.log(np.asarray(absA[np.arange(A.shape[0]), perm]).ravel()).sum()
    assert abs(lp - ref_lp) <= 1e-12 * max(1.0, abs(ref_lp)), (lp, ref_lp)


@pytest.mark.parametrize("seed", range(3))
def test_same_permutation_as_the_reference_on_a_unique_optimum(ref, seed):
    A = random_unsym(300, seed, spread=4.0)
    perm_r = hostlib.large_diag_perm(*csr_parts(A))[0]
    assert np.array_equal(perm_r, ref_ldperm(ref, A)[0])


@pytest.mark.parametrize("cplx", [False, True])
def test_equilibration_restatement_matches_dgsequ_dlaqgs(ref, cplx):
    """dgsequ_dist / dlaqgs_dist (zgsequ_dist / zlaqgs_dist) on a matrix with rows and columns scaled by 2^+-30: the same
    R, C, rowcnd, colcnd, amax and choice bit for bit"""
    rng = np.random.default_rng(5)
    A = sp.csr_matrix(random_unsym(200, 3, spread=2.0))
    n = A.shape[0]
    if cplx:
        A = sp.csr_matrix((A.data * np.exp(1j * rng.uniform(0, 6.3, A.nnz)), A.indices, A.indptr), shape=A.shape)
    A = sp.csr_matrix(sp.diags(np.exp2(rng.choice([-30.0, 0.0, 30.0], n))) @ A @ sp.diags(np.exp2(rng.choice([-30.0, 30.0], n))))
    rp, ci, v = csr_parts(A)
    one = np.ones(n)
    R, Cs, rowcnd, colcnd, amax, equed = equilibrate(rp, ci, v, one, one)
    Acsc = sp.csc_matrix(A)
    Acsc.sort_indices()
    nzval = np.ascontiguousarray(Acsc.data.astype(np.complex128 if cplx else np.float64))
    ri, cp = Acsc.indices.astype(np.int32), Acsc.indptr.astype(np.int32)
    store = _NC(len(ri), nzval.ctypes.data, ri.ctypes.data, cp.ctypes.data)
    M = _SuperMatrix(0, 3 if cplx else 1, 0, n, n, C.addressof(store))
    r, c = np.empty(n), np.empty(n)
    rc_, cc_, am = C.c_double(), C.c_double(), C.c_double()
    info = C.c_int(0)
    p = "z" if cplx else "d"
    getattr(ref, p + "gsequ_dist")(C.byref(M), r.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p), C.byref(rc_),
                                   C.byref(cc_), C.byref(am), C.byref(info))
    assert info.value == 0
    eq = C.create_string_buffer(1)
    laqgs = getattr(ref, p + "laqgs_dist")
    laqgs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_char_p]
    laqgs(C.addressof(M), r.ctypes.data, c.ctypes.data, rc_.value, cc_.value, am.value, eq)
    assert (rowcnd, colcnd, amax) == (rc_.value, cc_.value, am.value)
    assert "NRCB"[equed] == eq.value.decode()
    assert np.array_equal(R, r if equed & 1 else one) and np.array_equal(Cs, c if equed & 2 else one)
