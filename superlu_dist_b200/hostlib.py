"""ctypes binding of lib/libslu_b200_host.so (include/slu_b200_host.h): synthetic matrices,
geometric nested dissection, symbolic factorization into the reference's L/U block layout, Z-forest
partition and the panel mat-vec used by the ||LU - A|| checker.  Host-only (no CUDA)."""
import ctypes as C
import os

import numpy as np

from ._paths import HOST_SO

_lib = None

i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(HOST_SO):
        raise RuntimeError(
            f"{HOST_SO} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` first")
    L = C.CDLL(HOST_SO)
    L.sluh_poisson3d_nnz.restype = C.c_int64
    L.sluh_poisson3d_nnz.argtypes = [C.c_int] * 3
    L.sluh_poisson3d.argtypes = [C.c_int] * 3 + [i32p, i32p, f64p]
    L.sluh_fem3d_nnz.restype = C.c_int64
    L.sluh_fem3d_nnz.argtypes = [C.c_int] * 4
    L.sluh_fem3d.argtypes = [C.c_int] * 4 + [C.c_uint64, i32p, i32p, f64p]
    L.sluh_nd_order.argtypes = [C.c_int] * 5 + [i32p]
    L.sluh_nd_order_graph.restype = C.c_int
    L.sluh_nd_order_graph.argtypes = [C.c_int, i32p, i32p, C.c_int, C.c_int, i32p]
    L.sluh_symbolic.restype = C.c_void_p
    L.sluh_symbolic.argtypes = [C.c_int, i32p, i32p, C.c_void_p, C.c_int, C.c_int, C.c_double]
    L.sluh_symbolic_schur.restype = C.c_void_p
    L.sluh_symbolic_schur.argtypes = [C.c_int, i32p, i32p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int]
    L.sluh_symb_free.argtypes = [C.c_void_p]
    L.sluh_symb_nsupers.restype = C.c_int32
    L.sluh_symb_nsupers.argtypes = [C.c_void_p]
    L.sluh_symb_sizes.argtypes = [C.c_void_p, f64p]
    L.sluh_symb_export.argtypes = [C.c_void_p, i32p, i32p, i32p, i64p, i32p, i64p, i64p, i32p, i64p]
    L.sluh_fill_values.argtypes = [C.c_int, i32p, i32p, f64p, i32p, C.c_int, i32p, i64p, i32p, i64p,
                                   C.c_void_p, i64p, i32p, i64p, C.c_void_p, C.c_void_p]
    L.sluh_forests.argtypes = [C.c_int, i32p, f64p, C.c_int, i32p]
    L.sluh_panel_matvec.argtypes = [C.c_int, C.c_int, C.c_int, i32p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, f64p, f64p]
    L.sluh_read_matrix.restype = C.c_void_p
    L.sluh_read_matrix.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    L.sluh_matrix_dims.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]
    L.sluh_matrix_export_csc.argtypes = [C.c_void_p, i32p, i32p, f64p]
    L.sluh_matrix_export_csr.argtypes = [C.c_void_p, i32p, i32p, f64p]
    L.sluh_matrix_free.argtypes = [C.c_void_p]
    L.sluh_write_binary.argtypes = [C.c_char_p, C.c_int32, C.c_int32, i32p, i32p, f64p]
    L.sluh_large_diag_perm.argtypes = [C.c_int, i32p, i32p, f64p, i32p, f64p, f64p, f64p]
    _lib = L
    return L


def large_diag_perm(rowptr, colind, val):
    """Maximum-product matching with the MC64 job-5 scalings (sluh_large_diag_perm) -> (perm_r, R, C, logprod):
    perm_r[i] = the row of Pr A that holds row i of A, |R_i a_ij C_j| <= 1 with equality on the matching, logprod =
    sum_i log |a_{i, perm_r[i]}|.  val may be complex (the modulus is matched).  Raises ValueError, naming the
    structural rank, if A is structurally singular."""
    rp = np.ascontiguousarray(rowptr, np.int32)
    ci = np.ascontiguousarray(colind, np.int32)
    av = np.ascontiguousarray(np.abs(np.asarray(val)), np.float64)
    n = len(rp) - 1
    perm_r = np.empty(n, np.int32)
    R, Cs, out = np.empty(n), np.empty(n), np.zeros(2)
    rc = lib().sluh_large_diag_perm(n, rp, ci, av, perm_r, R, Cs, out)
    if rc < 0:
        raise ValueError("sluh_large_diag_perm: bad CSR input (rowptr, colind outside 0 .. n-1, or a non-finite value)")
    if rc > 0 or out[0] == -np.inf:
        raise ValueError(f"A is structurally singular: structural rank {rc} < n = {n}")
    return perm_r, R, Cs, float(out[0])


def row_permute(rowptr, colind, val, perm_r):
    """CSR of Pr A: row i of A becomes row perm_r[i] (columns and their order within a row kept)."""
    rp = np.asarray(rowptr, np.int64)
    ci, v = np.asarray(colind), np.asarray(val)
    perm_r = np.asarray(perm_r, np.int64)
    n = len(rp) - 1
    inv = np.empty(n, np.int64)
    inv[perm_r] = np.arange(n)
    cnt = np.diff(rp)[inv]
    nrp = np.concatenate([[0], np.cumsum(cnt)])
    src = np.repeat(rp[:-1][inv] - nrp[:-1], cnt) + np.arange(nrp[-1])
    return nrp.astype(np.int32), ci[src].astype(np.int32), v[src]


def read_matrix(path, fmt=None, layout="csr"):
    """Harwell-/Rutherford-Boeing, Matrix Market, triplet (.dat / .datnh) or reference-binary file -> (nrow, ncol, ptr, ind, val) in CSR (default) or CSC
    (the reference's dreadhb_dist / dreadMM_dist / dread_binary return CSC).  Complex files give complex128 values.
    Symmetric storage is expanded to the full matrix, as the reference's readers do."""
    L = lib()
    err = C.create_string_buffer(512)
    h = L.sluh_read_matrix(os.fsencode(path), fmt.encode() if fmt else None, err, 512)
    if not h:
        raise ValueError(f"read_matrix({path}): {err.value.decode()}")
    try:
        nr, nc, nnz, cx = C.c_int32(), C.c_int32(), C.c_int64(), C.c_int32()
        L.sluh_matrix_dims(h, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(cx))
        n_ptr = (nr.value if layout == "csr" else nc.value) + 1
        ptr = np.empty(n_ptr, np.int32)
        ind = np.empty(max(nnz.value, 1), np.int32)
        val = np.empty(max(nnz.value, 1) * (2 if cx.value else 1), np.float64)
        (L.sluh_matrix_export_csr if layout == "csr" else L.sluh_matrix_export_csc)(h, ptr, ind, val)
        ind = ind[:nnz.value]
        val = val[:nnz.value * (2 if cx.value else 1)]
        if cx.value:
            val = val.view(np.complex128)
        return nr.value, nc.value, ptr, ind, val
    finally:
        L.sluh_matrix_free(h)


def write_binary(path, n, colptr, rowind, val):
    """The reference's dwrite_binary layout (SRC/double/dbinary_io.c:24-42) at `path`."""
    rc = lib().sluh_write_binary(os.fsencode(path), n, len(rowind), np.ascontiguousarray(colptr, np.int32),
                                 np.ascontiguousarray(rowind, np.int32), np.ascontiguousarray(val, np.float64))
    if rc != 0:
        raise OSError(f"cannot write {path}")


def poisson3d(nx, ny=None, nz=None):
    """7-point Laplacian, Dirichlet, a_ii=6, a_ij=-1 (BASELINE.json configs[1]); CSR int32."""
    ny = nx if ny is None else ny
    nz = nx if nz is None else nz
    L = lib()
    n = nx * ny * nz
    nnz = L.sluh_poisson3d_nnz(nx, ny, nz)
    rowptr = np.empty(n + 1, np.int32)
    colind = np.empty(nnz, np.int32)
    val = np.empty(nnz, np.float64)
    L.sluh_poisson3d(nx, ny, nz, rowptr, colind, val)
    return rowptr, colind, val


def fem3d(nx, ny=None, nz=None, dof=3, seed=20260924):
    """audikw_1-shaped synthetic: dof unknowns per node, 27-point coupling (configs[2])."""
    ny = nx if ny is None else ny
    nz = nx if nz is None else nz
    L = lib()
    n = nx * ny * nz * dof
    nnz = L.sluh_fem3d_nnz(nx, ny, nz, dof)
    rowptr = np.empty(n + 1, np.int32)
    colind = np.empty(nnz, np.int32)
    val = np.empty(nnz, np.float64)
    L.sluh_fem3d(nx, ny, nz, dof, seed, rowptr, colind, val)
    return rowptr, colind, val


def nd_order(nx, ny=None, nz=None, dof=1, leaf=32):
    ny = nx if ny is None else ny
    nz = nx if nz is None else nz
    perm = np.empty(nx * ny * nz * dof, np.int32)
    lib().sluh_nd_order(nx, ny, nz, dof, leaf, perm)
    return perm


def nd_order_graph(rowptr, colind, leaf=64, compress_dof=True):
    """Nested dissection of a general sparse pattern (A + A^T): perm[old] = new.  For matrices without a geometry
    (read_matrix); the role of ColPerm = METIS_AT_PLUS_A in the reference (get_perm_c.c:479)."""
    rowptr = np.ascontiguousarray(rowptr, np.int32)
    colind = np.ascontiguousarray(colind, np.int32)
    n = len(rowptr) - 1
    perm = np.empty(n, np.int32)
    rc = lib().sluh_nd_order_graph(n, rowptr, colind, int(leaf), 1 if compress_dof else 0, perm)
    if rc:
        raise RuntimeError(f"sluh_nd_order_graph failed ({rc})")
    return perm


def schur_order(rowptr, colind, schur, leaf=64):
    """A fill-reducing ordering that numbers the Schur unknowns `schur` (distinct indices) last: nested dissection
    (nd_order_graph) of the pattern with their rows and columns removed, then schur[t] -> n - s + t.  perm[old] = new,
    for Symbolic / LUProblem.from_matrix with nschur = len(schur)."""
    rowptr = np.asarray(rowptr, np.int64)
    colind = np.asarray(colind, np.int64)
    n = len(rowptr) - 1
    schur = np.asarray(schur, np.int64)
    s = len(schur)
    if s > n or (s and (schur.min() < 0 or schur.max() >= n)) or len(np.unique(schur)) != s:
        raise ValueError("schur must hold distinct indices in [0, n)")
    keep = np.ones(n, bool)
    keep[schur] = False
    new_of = np.full(n, -1, np.int64)
    new_of[keep] = np.arange(n - s)
    perm = np.empty(n, np.int32)
    perm[schur] = np.arange(n - s, n)
    if n - s:
        rows = np.repeat(np.arange(n), np.diff(rowptr))
        m = keep[rows] & keep[colind]
        rp = np.concatenate([[0], np.cumsum(np.bincount(new_of[rows[m]], minlength=n - s))]).astype(np.int32)
        sub = nd_order_graph(rp, new_of[colind[m]].astype(np.int32), leaf)
        perm[keep] = sub
    return perm


class Symbolic:
    """Result of sluh_symbolic: supernode partition + L/U index arenas in the reference layout.  nschur > 0
    (sluh_symbolic_schur): the columns perm sends to n - nschur .. n - 1 stay last, in their order, and form whole
    supernodes -- the layout of a partial factorization (slu_b200_schur_create)."""

    def __init__(self, n, rowptr, colind, perm=None, relax=32, maxsup=256, amalg=0.05, nschur=0):
        L = lib()
        rowptr = np.ascontiguousarray(rowptr, np.int32)
        colind = np.ascontiguousarray(colind, np.int32)
        pp = None
        if perm is not None:
            perm = np.ascontiguousarray(perm, np.int32)
            pp = perm.ctypes.data_as(C.c_void_p)
        if nschur:
            h = L.sluh_symbolic_schur(n, rowptr, colind, pp, relax, maxsup, amalg, int(nschur))
            if not h:
                raise ValueError(f"nschur = {nschur} must lie in [0, n = {n}]")
        else:
            h = L.sluh_symbolic(n, rowptr, colind, pp, relax, maxsup, amalg)
        self.nschur = int(nschur)
        try:
            self.n = n
            self.nsupers = L.sluh_symb_nsupers(h)
            sz = np.zeros(8, np.float64)
            L.sluh_symb_sizes(h, sz)
            self.lidx_len, self.lval_len, self.uidx_len, self.uval_len = (int(s) for s in sz[:4])
            self.ops_fact, self.ops_schur = float(sz[4]), float(sz[5])
            ns = self.nsupers
            self.perm = np.empty(n, np.int32)
            self.xsup = np.empty(ns + 1, np.int32)
            self.setree = np.empty(ns, np.int32)
            self.lidx_off = np.empty(ns + 1, np.int64)
            self.lval_off = np.empty(ns + 1, np.int64)
            self.uidx_off = np.empty(ns + 1, np.int64)
            self.uval_off = np.empty(ns + 1, np.int64)
            self.lidx = np.empty(max(self.lidx_len, 1), np.int32)
            self.uidx = np.empty(max(self.uidx_len, 1), np.int32)
            L.sluh_symb_export(h, self.perm, self.xsup, self.setree, self.lidx_off, self.lidx,
                               self.lval_off, self.uidx_off, self.uidx, self.uval_off)
        finally:
            L.sluh_symb_free(h)


def forests(setree, weight, max_lvl):
    setree = np.ascontiguousarray(setree, np.int32)
    out = np.empty(len(setree), np.int32)
    lib().sluh_forests(len(setree), setree, np.ascontiguousarray(weight, np.float64), max_lvl, out)
    return out
