"""ctypes binding of lib/libslu_b200.so (include/slu_b200.h) -- the product's C-ABI.

There is no CPU fallback: if the shared library is missing, or no CUDA device is visible when a
compute entry point is called, this module raises.
"""
import ctypes as C
import os
import re

import numpy as np

from ._paths import CUDA_SO, INCLUDE
from .problem import my_tree_idxs, my_zero_tr_idxs

_lib = None
i32 = C.c_int32


class Forest(C.Structure):
    _fields_ = [("nNodes", i32), ("nodeList", C.c_void_p), ("numLvl", i32), ("eTreeTopLims", C.c_void_p)]


class LUView(C.Structure):
    _fields_ = [("n", i32), ("nsupers", i32), ("xsup", C.c_void_p),
                ("nprow", i32), ("npcol", i32), ("npdep", i32), ("myrow", i32), ("mycol", i32), ("mydep", i32),
                ("Lrowind_bc_ptr", C.c_void_p), ("Lnzval_bc_ptr", C.c_void_p),
                ("Ufstnz_br_ptr", C.c_void_p), ("Unzval_br_ptr", C.c_void_p),
                ("maxLvl", i32), ("myTreeIdxs", C.c_void_p), ("myZeroTrIdxs", C.c_void_p),
                ("nforests", i32), ("forests", C.c_void_p)]


class Options(C.Structure):
    _fields_ = [("device", i32), ("replace_tiny_pivot", i32), ("thresh", C.c_double), ("verbose", i32),
                ("pinned_host", i32), ("world_size", i32), ("world_rank", i32),
                ("nccl_id", C.c_ubyte * 128), ("schur_variant", i32), ("reserved", i32 * 7)]


class Stats(C.Structure):
    _fields_ = [("ops_fact", C.c_double), ("ops_schur", C.c_double), ("schur_bytes", C.c_double),
                ("tiny_pivots", C.c_int64), ("gpu_launches", C.c_int64),
                ("t_analyze_s", C.c_double), ("t_upload_s", C.c_double), ("t_factor_s", C.c_double),
                ("t_download_s", C.c_double), ("t_diag_ms", C.c_double), ("t_trsm_ms", C.c_double),
                ("t_schur_setup_ms", C.c_double), ("t_schur_ms", C.c_double), ("t_reduce_ms", C.c_double),
                ("lu_device_bytes", C.c_int64), ("index_device_bytes", C.c_int64),
                ("nnz_l", C.c_int64), ("nnz_u", C.c_int64), ("nlevels", i32), ("my_supernodes", i32),
                ("reserved", C.c_double * 8)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


def declared_symbols():
    """Every function declared in include/slu_b200.h."""
    text = open(os.path.join(INCLUDE, "slu_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b((?:slu_b200_|pdgstrf3d_b200|pzgstrf3d_b200)\w*)\s*\(", text)))


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(CUDA_SO):
        raise RuntimeError(f"{CUDA_SO} is missing: the CUDA extension was not built "
                           "(python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback")
    L = C.CDLL(CUDA_SO)
    for s in declared_symbols():
        if not hasattr(L, s):
            raise RuntimeError(f"libslu_b200.so does not export {s}")
    sizes = (i32 * 4)()
    L.slu_b200_struct_sizes(sizes)
    mine = [C.sizeof(Forest), C.sizeof(LUView), C.sizeof(Options), C.sizeof(Stats)]
    if list(sizes) != mine:
        raise RuntimeError(f"ctypes struct mirrors are out of date: library {list(sizes)} vs python {mine}")
    L.slu_b200_last_error.restype = C.c_char_p
    L.slu_b200_host_alloc.restype = C.c_void_p
    L.slu_b200_host_alloc.argtypes = [C.c_size_t]
    L.slu_b200_host_free.argtypes = [C.c_void_p]
    L.slu_b200_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(LUView), C.POINTER(Options)]
    for f in ("slu_b200_upload", "slu_b200_download"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.slu_b200_factor.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.slu_b200_factor_host.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.slu_b200_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
    L.slu_b200_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.slu_b200_fill_csr.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.slu_b200_destroy.argtypes = [C.c_void_p]
    L.slu_b200_destroy.restype = None
    L.pdgstrf3d_b200.argtypes = [C.POINTER(LUView), C.POINTER(Options), C.POINTER(Stats), C.POINTER(C.c_int)]
    L.slu_b200_plan.argtypes = [C.POINTER(LUView), C.POINTER(Options), C.POINTER(Stats)]
    L.slu_b200_z_plan.argtypes = [C.POINTER(LUView), C.POINTER(Options), C.POINTER(Stats)]
    # doublecomplex twins (same structs; value arrays hold (re, im) pairs)
    L.slu_b200_z_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(LUView), C.POINTER(Options)]
    for f in ("slu_b200_z_upload", "slu_b200_z_download"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.slu_b200_z_factor.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.slu_b200_z_factor_host.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.slu_b200_z_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
    L.slu_b200_z_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.slu_b200_z_fill_csr.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.slu_b200_z_destroy.argtypes = [C.c_void_p]
    L.slu_b200_z_destroy.restype = None
    L.pzgstrf3d_b200.argtypes = [C.POINTER(LUView), C.POINTER(Options), C.POINTER(Stats), C.POINTER(C.c_int)]
    # batched handles (many matrices of one pattern)
    L.slu_b200_batch_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(LUView), C.POINTER(Options), C.c_int]
    L.slu_b200_batch_fill_csr.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.slu_b200_batch_factor.argtypes = [C.c_void_p, C.c_void_p]
    L.slu_b200_batch_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.slu_b200_batch_download.argtypes = [C.c_void_p, C.c_int]
    L.slu_b200_z_batch_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(LUView), C.POINTER(Options), C.c_int]
    L.slu_b200_z_batch_fill_csr.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.slu_b200_z_batch_factor.argtypes = [C.c_void_p, C.c_void_p]
    L.slu_b200_z_batch_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.slu_b200_z_batch_download.argtypes = [C.c_void_p, C.c_int]
    for f in ("slu_b200_solve_trans", "slu_b200_z_solve_trans", "slu_b200_batch_solve_trans", "slu_b200_z_batch_solve_trans"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    for f in ("slu_b200_gscon", "slu_b200_z_gscon"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_char, C.c_double, C.POINTER(C.c_double)]
    for f in ("slu_b200_batch_gscon", "slu_b200_z_batch_gscon"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_char, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_selinv", "slu_b200_z_selinv"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p]
    for f in ("slu_b200_selinv_get", "slu_b200_z_selinv_get"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_logdet", "slu_b200_z_logdet"):
        getattr(L, f).argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_void_p]
    for f in ("slu_b200_batch_selinv", "slu_b200_z_batch_selinv"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p]
    for f in ("slu_b200_batch_selinv_get", "slu_b200_z_batch_selinv_get"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_batch_logdet", "slu_b200_z_batch_logdet"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_inertia", "slu_b200_z_inertia"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
    for f in ("slu_b200_batch_inertia", "slu_b200_z_batch_inertia"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_batch_fill_affine", "slu_b200_z_batch_fill_affine"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_schur_create", "slu_b200_z_schur_create"):
        getattr(L, f).argtypes = [C.POINTER(C.c_void_p), C.POINTER(LUView), C.POINTER(Options), C.c_int]
    for f in ("slu_b200_schur_get", "slu_b200_z_schur_get"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    for f in ("slu_b200_schur_condense", "slu_b200_z_schur_condense", "slu_b200_schur_expand", "slu_b200_z_schur_expand"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    for f in ("slu_b200_batch_schur_create", "slu_b200_z_batch_schur_create"):
        getattr(L, f).argtypes = [C.POINTER(C.c_void_p), C.POINTER(LUView), C.POINTER(Options), C.c_int, C.c_int]
    for f in ("slu_b200_batch_schur_get", "slu_b200_z_batch_schur_get"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    for f in ("slu_b200_batch_schur_condense", "slu_b200_z_batch_schur_condense", "slu_b200_batch_schur_expand",
              "slu_b200_z_batch_schur_expand"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    for f in ("slu_b200_fill_csr_scaled", "slu_b200_z_fill_csr_scaled"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7 + [C.c_int, C.c_void_p]
    for f in ("slu_b200_batch_fill_csr_scaled", "slu_b200_z_batch_fill_csr_scaled"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7 + [C.c_int, C.c_int, C.c_void_p]
    for f in ("slu_b200_get_scaling", "slu_b200_z_get_scaling"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_batch_get_scaling", "slu_b200_z_batch_get_scaling"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    for f in ("slu_b200_solve_scaled", "slu_b200_z_solve_scaled", "slu_b200_batch_solve_scaled", "slu_b200_z_batch_solve_scaled"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    _lib = L
    return L


def _is_complex(x):
    return np.dtype(x).kind == "c"


def _fn(name, complex_):
    """The double or the doublecomplex entry point: slu_b200_<name> / slu_b200_z_<name>."""
    return getattr(lib(), ("slu_b200_z_" if complex_ else "slu_b200_") + name)


def _check(rc):
    if rc != 0:
        raise RuntimeError("libslu_b200: " + lib().slu_b200_last_error().decode())


_TRANS = {"N": 0, "T": 1, "H": 2}   # the reference's trans_t: NOTRANS, TRANS, CONJ


def _solve_call(name, complex_, trans):
    """The solve entry point for trans 'N' | 'T' | 'H' (as SciPy's SuperLU.solve): (function, extra arguments).  'N' is
    the plain call (slu_b200_<name>), the others the _trans twin; 'H' of a real problem is 'T'."""
    if trans not in _TRANS:
        raise ValueError(f"trans must be 'N', 'T' or 'H', not {trans!r}")
    if trans == "N":
        return _fn(name, complex_), ()
    return _fn(name + "_trans", complex_), (_TRANS[trans],)


def _norm_byte(norm):
    """'1' | 'O' | 'I' (as LAPACK's gecon; lower case too) -> the char argument of slu_b200_gscon, which checks the letter"""
    if not (isinstance(norm, str) and len(norm) == 1 and norm.isascii()):
        raise ValueError(f"norm must be '1', 'O' or 'I', not {norm!r}")
    return norm.encode()


FILL_EQUIL = 1                      # SLU_B200_FILL_EQUIL
_SCALED_OUT = ("rowcnd", "colcnd", "amax", "equed", "norm_inf", "max_abs")


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _scaled_args(rowptr, colind, perm, perm_r, R, C_, rc_shape):
    """The int32 / float64 arrays of a scaled fill (None stays None: identity or ones)"""
    rp = np.ascontiguousarray(rowptr, np.int32)
    ci = np.ascontiguousarray(colind, np.int32)
    pm = np.ascontiguousarray(perm, np.int32)
    pr = None if perm_r is None else np.ascontiguousarray(perm_r, np.int32)
    sc = []
    for name, v in (("R", R), ("C", C_)):
        if v is not None:
            v = np.ascontiguousarray(v, np.float64)
            if v.shape not in rc_shape:
                raise ValueError(f"{name} must have shape {' or '.join(map(str, rc_shape))}, not {v.shape}")
        sc.append(v)
    return rp, ci, pm, pr, sc[0], sc[1]


def device_count():
    return lib().slu_b200_device_count()


def require_gpu():
    if device_count() < 1:
        raise RuntimeError("libslu_b200 needs a CUDA device; there is no CPU fallback")


def pinned_alloc(nbytes):
    """alloc(nbytes) -> (address, keepalive) for LUProblem.add_layer(alloc=...)."""
    L = lib()
    p = L.slu_b200_host_alloc(nbytes)
    if not p:
        raise MemoryError(f"cudaHostAlloc({nbytes}) failed")

    class _Keep:
        def __init__(self, p):
            self.p = p

        def __del__(self):
            try:
                L.slu_b200_host_free(self.p)
            except Exception:
                pass
    return p, _Keep(p)


def make_view(prob, z):
    """Fill a slu_b200_lu_view_t from an LUProblem layer; returns (view, keepalive)."""
    lay = prob.layers[z]
    li, lv, ui, uv = prob.pointer_tables(lay)
    trees = my_tree_idxs(prob.npdep, z)
    zeros = my_zero_tr_idxs(prob.npdep, z)
    nf = (1 << prob.max_lvl) - 1
    forests = (Forest * nf)()
    lims = []
    for f in range(nf):
        nodes = prob.forest_nodes[f]
        forests[f].nNodes = len(nodes)
        forests[f].nodeList = nodes.ctypes.data
        lim = np.array([0, len(nodes)], np.int32)
        lims.append(lim)
        forests[f].numLvl = 1
        forests[f].eTreeTopLims = lim.ctypes.data
    v = LUView()
    v.n, v.nsupers, v.xsup = prob.n, prob.nsupers, prob.xsup.ctypes.data
    v.nprow = v.npcol = 1
    v.npdep = prob.npdep
    v.myrow = v.mycol = 0
    v.mydep = z
    v.Lrowind_bc_ptr, v.Lnzval_bc_ptr = li.ctypes.data, lv.ctypes.data
    v.Ufstnz_br_ptr, v.Unzval_br_ptr = ui.ctypes.data, uv.ctypes.data
    v.maxLvl, v.myTreeIdxs, v.myZeroTrIdxs = prob.max_lvl, trees.ctypes.data, zeros.ctypes.data
    v.nforests, v.forests = nf, C.addressof(forests)
    return v, (li, lv, ui, uv, trees, zeros, forests, lims, lay)


def make_view_2d(prob, local, z):
    """View of the pieces process (local.myrow, local.mycol) of layer z holds (problem.Local2D)."""
    v, keep = make_view(prob, z)
    li, lv, ui, uv = local.pointer_tables()
    v.nprow, v.npcol, v.myrow, v.mycol = local.nprow, local.npcol, local.myrow, local.mycol
    v.Lrowind_bc_ptr, v.Lnzval_bc_ptr = li.ctypes.data, lv.ctypes.data
    v.Ufstnz_br_ptr, v.Unzval_br_ptr = ui.ctypes.data, uv.ctypes.data
    return v, (keep, li, lv, ui, uv, local)


def pdgstrf3d_2d(prob, local, z, **opt):
    """pdgstrf3d_b200 on a Pr x Pc x Pz grid: factor my pieces in place.  -> (info, Stats)"""
    require_gpu()
    view, keep = make_view_2d(prob, local, z)
    o = make_options(prob, **opt)
    st, info = Stats(), C.c_int(0)
    fn = lib().pzgstrf3d_b200 if _is_complex(prob.dtype) else lib().pdgstrf3d_b200   # complex16 twin: pzgstrf3d.c:120
    _check(fn(C.byref(view), C.byref(o), C.byref(st), C.byref(info)))
    del keep
    return info.value, st


def make_options(prob, device=-1, verbose=0, world_size=1, world_rank=0, nccl_id=None, pinned=0, schur_variant=0,
                 no_lookahead=0, no_coop=0, pipeline=0, overlap_h2d=0, tc_slices=0, tc_min_ns=0):
    o = Options()
    o.device = device
    o.replace_tiny_pivot = int(prob.replace_tiny_pivot)
    o.thresh = float(prob.thresh)
    o.verbose = verbose
    o.pinned_host = pinned
    o.schur_variant = schur_variant
    o.reserved[0] = no_lookahead   # 1: single-stream level loop (no overlap of panel work with the bulk update)
    o.reserved[2] = pipeline       # 1: pdgstrf3d_b200 overlaps H2D / factor / D2H (slu_b200_factor_host)
    o.reserved[1] = no_coop        # 1: reference-style ancestors (owner layer factors alone after a pairwise reduce)
    o.reserved[3] = overlap_h2d    # 1: level-by-level arena; factor_host also overlaps the upload (opt-in, DESIGN 9)
    o.reserved[4] = tc_slices      # int8 tensor-core path: int8 slices per operand (0 default: off, < 0 off, 5..8)
    o.reserved[5] = tc_min_ns      # narrowest supernode on the int8 tensor-core path (0: default)
    o.world_size, o.world_rank = world_size, world_rank
    if nccl_id is not None:
        C.memmove(o.nccl_id, bytes(nccl_id), 128)
    return o


def plan(prob, z=0, **opt):
    """slu_b200_plan / slu_b200_z_plan: the analysis of layer z without a device -> Stats (HBM bytes, flops ...)."""
    view, keep = make_view(prob, z)
    o = make_options(prob, **opt)
    st = Stats()
    _check(_fn("plan", _is_complex(prob.dtype))(C.byref(view), C.byref(o), C.byref(st)))
    del keep
    return st


def nccl_unique_id():
    buf = (C.c_ubyte * 128)()
    _check(lib().slu_b200_nccl_unique_id(buf))
    return bytes(buf)


class Handle:
    """slu_b200_handle_t: create (analysis + HBM allocation) / upload / factor / download."""

    def __init__(self, prob, z=0, **opt):
        require_gpu()
        self.prob = prob
        self.z_ = _is_complex(prob.dtype)     # doublecomplex problem -> slu_b200_z_* (pzgstrf3d)
        self.view, self._keep = make_view(prob, z)
        self.opt = make_options(prob, **opt)
        self.h = C.c_void_p()
        _check(_fn("create", self.z_)(C.byref(self.h), C.byref(self.view), C.byref(self.opt)))

    def upload(self):
        _check(_fn("upload", self.z_)(self.h))

    def factor(self):
        info = C.c_int(0)
        _check(_fn("factor", self.z_)(self.h, C.byref(info)))
        return info.value

    def factor_host(self):
        """upload + factor + download with the transfers overlapped (slu_b200_factor_host)."""
        info = C.c_int(0)
        _check(_fn("factor_host", self.z_)(self.h, C.byref(info)))
        return info.value

    def download(self):
        _check(_fn("download", self.z_)(self.h))

    def fill_csr(self, rowptr, colind, val, perm):
        """Device-side distribution (slu_b200_fill_csr): P A P^T scattered into the HBM panels by a kernel; replaces
        upload().  perm[old] = new.  val is complex128 for a complex problem (slu_b200_z_fill_csr)."""
        rp = np.ascontiguousarray(rowptr, np.int32)
        ci = np.ascontiguousarray(colind, np.int32)
        v = np.ascontiguousarray(val, self._dtype())
        pm = np.ascontiguousarray(perm, np.int32)
        _check(_fn("fill_csr", self.z_)(self.h, len(rp) - 1, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                                        v.ctypes.data_as(C.c_void_p), pm.ctypes.data_as(C.c_void_p)))

    def fill_csr_scaled(self, rowptr, colind, val, perm, perm_r=None, R=None, C=None, equil=True):
        """Scaled, row-permuted device fill (slu_b200_fill_csr_scaled): F = Pc Pr Dr A Dc Pc^T, entry (i, j) of A to
        F(perm[perm_r[i]], perm[j]) as (R[i] a_ij) C[j]; perm_r, R, C from hostlib.large_diag_perm (None: identity / ones),
        perm the ordering of the pattern of Pr A.  equil: equilibrate Pr Dr A Dc on the device (dgsequ / dlaqgs) and fold the
        factors into R and C.  Replaces upload().  -> dict rowcnd, colcnd, amax, equed (0 none, 1 rows, 2 columns, 3 both),
        norm_inf (||F||_inf, for rcond(norm_inf, 'I')), max_abs"""
        rp, ci, pm, pr, Rv, Cv = _scaled_args(rowptr, colind, perm, perm_r, R, C, [(self.prob.n,)])
        v = np.ascontiguousarray(val, self._dtype())
        out = np.zeros(6)
        _check(_fn("fill_csr_scaled", self.z_)(self.h, len(rp) - 1, _ptr(rp), _ptr(ci), _ptr(v), _ptr(pr), _ptr(pm), _ptr(Rv),
                                               _ptr(Cv), FILL_EQUIL if equil else 0, _ptr(out)))
        return {k: (int(x) if k == "equed" else float(x)) for k, x in zip(_SCALED_OUT, out)}

    def scaling(self):
        """(perm_r, R, C) of the last scaled fill, R and C with the equilibration folded in (slu_b200_get_scaling)"""
        n = self.prob.n
        pr, Rv, Cv = np.empty(n, np.int32), np.empty(n), np.empty(n)
        _check(_fn("get_scaling", self.z_)(self.h, _ptr(pr), _ptr(Rv), _ptr(Cv)))
        return pr, Rv, Cv

    def solve_scaled(self, b, trans="N"):
        """op(A) x = b in A's own ordering on the factors of a scaled fill (slu_b200_solve_scaled): the row permutation,
        the scalings and perm are applied on the device.  b: (n,) or (nrhs, n); trans 'N', 'T' or 'H'."""
        if trans not in _TRANS:
            raise ValueError(f"trans must be 'N', 'T' or 'H', not {trans!r}")
        x = np.array(b, self._dtype(), order="C", copy=True)
        nrhs = 1 if x.ndim == 1 else x.shape[0]
        _check(_fn("solve_scaled", self.z_)(self.h, _ptr(x), self.prob.n, nrhs, _TRANS[trans]))
        return x

    def solve(self, b, trans="N"):
        """L U x = b on the device-resident factors (slu_b200_solve / slu_b200_z_solve); b: (n,) or (nrhs, n), ordering
        of the factored matrix, complex128 for a complex problem.  Returns x with the same shape and dtype.
        trans = 'T' solves A^T x = b, 'H' A^H x = b (slu_b200_solve_trans / slu_b200_z_solve_trans) on the same factors."""
        fn, extra = _solve_call("solve", self.z_, trans)
        x = np.array(b, self._dtype(), order="C", copy=True)
        nrhs = 1 if x.ndim == 1 else x.shape[0]
        _check(fn(self.h, x.ctypes.data_as(C.c_void_p), self.prob.n, nrhs, *extra))
        return x

    def rcond(self, anorm, norm="1"):
        """Reciprocal condition number estimate on the resident factors (slu_b200_gscon / slu_b200_z_gscon), as LAPACK's
        gecon: (1 / est ||F^-1||) / anorm with anorm = ||A|| in the same norm, '1' (or 'O') or 'I'."""
        out = C.c_double(0.0)
        _check(_fn("gscon", self.z_)(self.h, _norm_byte(norm), float(anorm), C.byref(out)))
        return out.value

    def selinv(self):
        """Selected inversion on the resident factors (slu_b200_selinv / slu_b200_z_selinv): H = F^-T on the pattern of
        L + U (a plain transpose in complex too), kept in HBM for inv_entries / inv_diag.  -> (seconds, flops, kernel
        launches, HBM bytes held); in complex the flops count a complex multiply-add as 2, as ops_fact does."""
        out = (C.c_double * 4)()
        _check(_fn("selinv", self.z_)(self.h, out))
        return tuple(out)

    def inv_entries(self, rowptr, colind, perm):
        """(A^-1)(i, colind[p]) for every entry p of row i of a CSR pattern (slu_b200_selinv_get), perm[old] = new as in
        fill_csr; every entry must have a slot in L + U.  -> float64 (complex128 for a complex problem) array (nnz,)"""
        rp = np.ascontiguousarray(rowptr, np.int32)
        ci = np.ascontiguousarray(colind, np.int32)
        pm = np.ascontiguousarray(perm, np.int32)
        out = np.empty(len(ci), self._dtype())
        _check(_fn("selinv_get", self.z_)(self.h, len(rp) - 1, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                                          pm.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        return out

    def inv_diag(self, perm=None):
        """The diagonal of A^-1 (perm[old] = new; None: the identity, i.e. the diagonal of F^-1)."""
        n = self.prob.n
        pm = np.arange(n, dtype=np.int32) if perm is None else perm
        return self.inv_entries(np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32), pm)

    def logdet(self):
        """(sign, log |det A|) from the resident factors (slu_b200_logdet / slu_b200_z_logdet), as numpy.linalg.slogdet:
        the sign is a float +-1, or for a complex problem a complex128 of modulus 1"""
        la, sg = C.c_double(0.0), np.zeros(2 if self.z_ else 1, np.float64)
        _check(_fn("logdet", self.z_)(self.h, C.byref(la), sg.ctypes.data_as(C.c_void_p)))
        return (complex(sg[0], sg[1]) if self.z_ else float(sg[0])), la.value

    def inertia(self):
        """Inertia of a symmetric (Hermitian) A from the signs of the resident pivots (slu_b200_inertia / slu_b200_z_inertia)
        -> (neg, pos, tiny, defect): the pivots with Re u_ii < 0, the others (neg + pos = n), those with |u_ii| <= thresh,
        and max |Im u_ii| / |u_ii| (0.0 for a real problem).  For A - sigma B with B positive definite, neg is the number
        of eigenvalues below sigma."""
        cnt, dfc = np.zeros(3, np.int64), C.c_double(0.0)
        _check(_fn("inertia", self.z_)(self.h, cnt.ctypes.data_as(C.c_void_p), C.byref(dfc)))
        return int(cnt[0]), int(cnt[1]), int(cnt[2]), dfc.value

    def _dtype(self):
        return np.complex128 if self.z_ else np.float64

    def stats(self):
        s = Stats()
        _check(_fn("get_stats", self.z_)(self.h, C.byref(s)))
        return s

    def close(self):
        if self.h:
            _fn("destroy", self.z_)(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SchurHandle(Handle):
    """A partial factorization (slu_b200_schur_create / slu_b200_z_schur_create): eliminate all unknowns of `prob` (layer 0,
    1 x 1 x 1 grid) but the last `nschur`, which must form whole supernodes (LUProblem.from_matrix(..., nschur=...)).
    upload / fill_csr / factor / download as Handle; schur() returns S = A22 - A21 A11^-1 A12, condense / expand the two
    partial solves.  Every other call of Handle fails on it.  A complex128 `prob` takes the doublecomplex twins."""

    def __init__(self, prob, nschur, **opt):
        require_gpu()
        self.prob, self.nschur = prob, int(nschur)
        self.z_ = _is_complex(prob.dtype)
        self.view, self._keep = make_view(prob, 0)
        self.opt = make_options(prob, **opt)
        self.h = C.c_void_p()
        _check(_fn("schur_create", self.z_)(C.byref(self.h), C.byref(self.view), C.byref(self.opt), self.nschur))

    def schur(self):
        """S (s, s), float64 or complex128: row / column t is unknown n - s + t of the factored ordering; exactly 0 off
        the stored pattern."""
        s = self.nschur
        out = np.empty((s, s), self._dtype(), order="F")
        _check(_fn("schur_get", self.z_)(self.h, out.ctypes.data_as(C.c_void_p), s))
        return out

    def _pass(self, name, b):
        x = np.array(b, self._dtype(), order="C", copy=True)
        nrhs = 1 if x.ndim == 1 else x.shape[0]
        _check(_fn(name, self.z_)(self.h, x.ctypes.data_as(C.c_void_p), self.prob.n, nrhs))
        return x

    def condense(self, b):
        """b: (n,) or (nrhs, n) in the factored ordering -> y1 = L11^-1 b1 in the eliminated positions, g = b2 - A21 A11^-1 b1
        in the last s"""
        return self._pass("schur_condense", b)

    def expand(self, y):
        """y: condense's result with x2 in the last s positions -> x1 = A11^-1 (b1 - A12 x2) there, x2 kept"""
        return self._pass("schur_expand", y)


class BatchHandle:
    """A batched handle (slu_b200_batch_*): `batch` matrices with the sparsity pattern of `prob` (layer 0, 1 x 1 x 1
    grid), factored and solved together.  The analysis is shared; each member has its own values.  A complex128 `prob`
    takes the doublecomplex twins (slu_b200_z_batch_*): values, right-hand sides and solutions are then complex128."""

    def __init__(self, prob, batch, **opt):
        require_gpu()
        self.prob, self.batch = prob, int(batch)
        self.z_ = _is_complex(prob.dtype)
        self.view, self._keep = make_view(prob, 0)
        self.opt = make_options(prob, **opt)
        self.h = C.c_void_p()
        _check(_fn("batch_create", self.z_)(C.byref(self.h), C.byref(self.view), C.byref(self.opt), self.batch))

    def _dtype(self):
        return np.complex128 if self.z_ else np.float64

    def fill_csr(self, rowptr, colind, vals, perm):
        """One CSR pattern and perm[old] = new for every member; vals: (batch, nnz), row j = member j's values."""
        rp = np.ascontiguousarray(rowptr, np.int32)
        ci = np.ascontiguousarray(colind, np.int32)
        v = np.ascontiguousarray(vals, self._dtype())
        if v.shape != (self.batch, len(ci)):
            raise ValueError(f"vals must have shape ({self.batch}, {len(ci)}), not {v.shape}")
        pm = np.ascontiguousarray(perm, np.int32)
        _check(_fn("batch_fill_csr", self.z_)(self.h, len(rp) - 1, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                                              v.ctypes.data_as(C.c_void_p), pm.ctypes.data_as(C.c_void_p)))

    def fill_csr_scaled(self, rowptr, colind, vals, perm, perm_r=None, R=None, C=None, equil=True):
        """Handle.fill_csr_scaled for every member (slu_b200_batch_fill_csr_scaled): one pattern, perm_r and perm; vals
        (batch, nnz); R and C (n,) shared or (batch, n) per member.  The equilibration runs per member.  -> dict of float64
        arrays (batch,) with the keys of Handle.fill_csr_scaled (equed int32)"""
        n, B = self.prob.n, self.batch
        rp, ci, pm, pr, Rv, Cv = _scaled_args(rowptr, colind, perm, perm_r, R, C, [(n,), (B, n)])
        per = [x.ndim == 2 for x in (Rv, Cv) if x is not None]
        if len(set(per)) > 1:
            raise ValueError("R and C must both be shared (n,) or both per member (batch, n)")
        v = np.ascontiguousarray(vals, self._dtype())
        if v.shape != (B, len(ci)):
            raise ValueError(f"vals must have shape ({B}, {len(ci)}), not {v.shape}")
        out = np.zeros((B, 6))
        _check(_fn("batch_fill_csr_scaled", self.z_)(self.h, len(rp) - 1, _ptr(rp), _ptr(ci), _ptr(v), _ptr(pr), _ptr(pm), _ptr(Rv),
                                                     _ptr(Cv), int(bool(per and per[0])), FILL_EQUIL if equil else 0, _ptr(out)))
        res = {k: out[:, t].copy() for t, k in enumerate(_SCALED_OUT)}
        res["equed"] = res["equed"].astype(np.int32)
        return res

    def scaling(self, member):
        """(R, C) of member `member` after the last scaled fill (slu_b200_batch_get_scaling)"""
        n = self.prob.n
        Rv, Cv = np.empty(n), np.empty(n)
        _check(_fn("batch_get_scaling", self.z_)(self.h, int(member), _ptr(Rv), _ptr(Cv)))
        return Rv, Cv

    def solve_scaled(self, b, trans="N"):
        """Handle.solve_scaled for every member (slu_b200_batch_solve_scaled); b: (batch, n) or (batch, nrhs, n) in A's
        ordering"""
        if trans not in _TRANS:
            raise ValueError(f"trans must be 'N', 'T' or 'H', not {trans!r}")
        x = np.array(b, self._dtype(), order="C", copy=True)
        if x.ndim not in (2, 3) or x.shape[0] != self.batch or x.shape[-1] != self.prob.n:
            raise ValueError(f"b must have shape ({self.batch}, n) or ({self.batch}, nrhs, n) with n = {self.prob.n}")
        nrhs = 1 if x.ndim == 2 else x.shape[1]
        _check(_fn("batch_solve_scaled", self.z_)(self.h, _ptr(x), self.prob.n, nrhs, _TRANS[trans]))
        return x

    def factor(self):
        """-> int32 array (batch,): 0, or the 1-based column of the member's first exact zero pivot."""
        info = np.zeros(self.batch, np.int32)
        _check(_fn("batch_factor", self.z_)(self.h, info.ctypes.data_as(C.c_void_p)))
        return info

    def solve(self, b, trans="N"):
        """L_j U_j x_j = b_j for every member; b: (batch, n) or (batch, nrhs, n), ordering of the factored matrix.
        trans = 'T' / 'H' solves A_j^T x_j = b_j / A_j^H x_j = b_j (slu_b200_batch_solve_trans)."""
        fn, extra = _solve_call("batch_solve", self.z_, trans)
        x = np.array(b, self._dtype(), order="C", copy=True)
        if x.ndim not in (2, 3) or x.shape[0] != self.batch or x.shape[-1] != self.prob.n:
            raise ValueError(f"b must have shape ({self.batch}, n) or ({self.batch}, nrhs, n) with n = {self.prob.n}")
        nrhs = 1 if x.ndim == 2 else x.shape[1]
        _check(fn(self.h, x.ctypes.data_as(C.c_void_p), self.prob.n, nrhs, *extra))
        return x

    def rcond(self, anorm, norm="1"):
        """Every member's reciprocal condition number estimate (slu_b200_batch_gscon), as Handle.rcond; anorm: (batch,)
        norms of the members, or one value for all.  -> float64 array (batch,)"""
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(anorm, np.float64), (self.batch,)))
        out = np.zeros(self.batch, np.float64)
        _check(_fn("batch_gscon", self.z_)(self.h, _norm_byte(norm), a.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        return out

    def selinv(self):
        """Selected inversion of every member (slu_b200_batch_selinv / slu_b200_z_batch_selinv), as Handle.selinv, kept in
        HBM for inv_entries / inv_diag.  -> (seconds, flops of all members, kernel launches, HBM bytes held); the launches
        are those of one unbatched sweep whatever the batch."""
        out = (C.c_double * 4)()
        _check(_fn("batch_selinv", self.z_)(self.h, out))
        return tuple(out)

    def inv_entries(self, rowptr, colind, perm):
        """(A_j^-1)(i, colind[p]) for every member j and every entry p of row i of one CSR pattern
        (slu_b200_batch_selinv_get), perm[old] = new as in fill_csr.  -> float64 (complex128) array (batch, nnz)"""
        rp = np.ascontiguousarray(rowptr, np.int32)
        ci = np.ascontiguousarray(colind, np.int32)
        pm = np.ascontiguousarray(perm, np.int32)
        out = np.empty((self.batch, len(ci)), self._dtype())
        _check(_fn("batch_selinv_get", self.z_)(self.h, len(rp) - 1, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                                                pm.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        return out

    def inv_diag(self, perm=None):
        """The diagonal of every member's A_j^-1 (perm as Handle.inv_diag).  -> (batch, n)"""
        n = self.prob.n
        pm = np.arange(n, dtype=np.int32) if perm is None else perm
        return self.inv_entries(np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32), pm)

    def logdet(self):
        """(sign, log |det A_j|) of every member (slu_b200_batch_logdet), as numpy.linalg.slogdet of a stack: sign (batch,)
        float64 of +-1, or complex128 of modulus 1 for a complex problem; logabs (batch,) float64"""
        la = np.zeros(self.batch, np.float64)
        sg = np.zeros(self.batch, np.complex128 if self.z_ else np.float64)
        _check(_fn("batch_logdet", self.z_)(self.h, la.ctypes.data_as(C.c_void_p), sg.ctypes.data_as(C.c_void_p)))
        return sg, la

    def inertia(self):
        """Every member's inertia (slu_b200_batch_inertia), as Handle.inertia -> (neg, pos, tiny, defect): int64 arrays
        (batch,) and a float64 array (batch,)"""
        cnt, dfc = np.zeros((self.batch, 3), np.int64), np.zeros(self.batch, np.float64)
        _check(_fn("batch_inertia", self.z_)(self.h, cnt.ctypes.data_as(C.c_void_p), dfc.ctypes.data_as(C.c_void_p)))
        return cnt[:, 0].copy(), cnt[:, 1].copy(), cnt[:, 2].copy(), dfc

    def fill_affine(self, rowptr, colind, terms, coef, perm):
        """An affine family on one CSR pattern (slu_b200_batch_fill_affine): member j's values are
        sum_t coef[j, t] * terms[t], computed on the device.  terms: (T, nnz), coef: (batch, T), float64 (complex128 for a
        complex problem); perm[old] = new as in fill_csr."""
        rp = np.ascontiguousarray(rowptr, np.int32)
        ci = np.ascontiguousarray(colind, np.int32)
        tv = np.ascontiguousarray(terms, self._dtype())
        cv = np.ascontiguousarray(coef, self._dtype())
        if tv.ndim != 2 or tv.shape[1] != len(ci):
            raise ValueError(f"terms must have shape (T, {len(ci)}), not {tv.shape}")
        if cv.shape != (self.batch, tv.shape[0]):
            raise ValueError(f"coef must have shape ({self.batch}, {tv.shape[0]}), not {cv.shape}")
        pm = np.ascontiguousarray(perm, np.int32)
        _check(_fn("batch_fill_affine", self.z_)(self.h, len(rp) - 1, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                                                 tv.shape[0], tv.ctypes.data_as(C.c_void_p), cv.ctypes.data_as(C.c_void_p),
                                                 pm.ctypes.data_as(C.c_void_p)))

    def download(self, member):
        """Member `member`'s L and U into prob.layers[0] (the reference layout)."""
        _check(_fn("batch_download", self.z_)(self.h, int(member)))

    def stats(self):
        s = Stats()
        _check(_fn("get_stats", self.z_)(self.h, C.byref(s)))
        return s

    def close(self):
        if self.h:
            _fn("destroy", self.z_)(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchSchurHandle(BatchHandle):
    """A partial factorization of `batch` matrices with the pattern of `prob` (slu_b200_batch_schur_create /
    slu_b200_z_batch_schur_create): as SchurHandle for every member, with the values, info and downloads of BatchHandle.
    fill_csr / fill_affine / factor / download as BatchHandle; schur() returns every member's S, condense / expand the two
    partial solves.  solve, rcond, selinv, inv_entries, inv_diag, logdet and inertia fail on it."""

    def __init__(self, prob, batch, nschur, **opt):
        require_gpu()
        self.prob, self.batch, self.nschur = prob, int(batch), int(nschur)
        self.z_ = _is_complex(prob.dtype)
        self.view, self._keep = make_view(prob, 0)
        self.opt = make_options(prob, **opt)
        self.h = C.c_void_p()
        _check(_fn("batch_schur_create", self.z_)(C.byref(self.h), C.byref(self.view), C.byref(self.opt), self.batch,
                                                  self.nschur))

    def schur(self, out=None):
        """(batch, s, s), float64 or complex128: [j] = S_j, row / column t is unknown n - s + t of the factored ordering;
        exactly 0 off the stored pattern.  out: a C-contiguous (batch, s, s) array of that dtype to write into instead of a
        new one (batch x s^2 values: reusing a buffer saves the page faults of fresh host memory on every call)."""
        s = self.nschur
        shape = (self.batch, s, s)
        if out is None:
            out = np.empty(shape, self._dtype())
        elif out.shape != shape or out.dtype != self._dtype() or not out.flags.c_contiguous:
            raise ValueError(f"out must be a C-contiguous {np.dtype(self._dtype()).name} array of shape {shape}")
        # member j's block is s x s column-major at j * s * s: a C-ordered (batch, s, s) array holds S_j^T in out[j]
        _check(_fn("batch_schur_get", self.z_)(self.h, out.ctypes.data_as(C.c_void_p), s))
        return out.transpose(0, 2, 1)

    def _pass(self, name, b):
        x = np.array(b, self._dtype(), order="C", copy=True)
        if x.ndim not in (2, 3) or x.shape[0] != self.batch or x.shape[-1] != self.prob.n:
            raise ValueError(f"b must have shape ({self.batch}, n) or ({self.batch}, nrhs, n) with n = {self.prob.n}")
        nrhs = 1 if x.ndim == 2 else x.shape[1]
        _check(_fn(name, self.z_)(self.h, x.ctypes.data_as(C.c_void_p), self.prob.n, nrhs))
        return x

    def condense(self, b):
        """b: (batch, n) or (batch, nrhs, n), as SchurHandle.condense for every member"""
        return self._pass("batch_schur_condense", b)

    def expand(self, y):
        """y: condense's result with x2 in the last s positions of every member, as SchurHandle.expand"""
        return self._pass("batch_schur_expand", y)


def pdgstrf3d(prob, z=0, **opt):
    """The one-call drop-in (pdgstrf3d_b200): factor layer z of `prob` in place.  -> (info, Stats)"""
    require_gpu()
    if _is_complex(prob.dtype):
        raise TypeError("pdgstrf3d is the double entry point; use pzgstrf3d for a complex128 problem")
    view, keep = make_view(prob, z)
    o = make_options(prob, **opt)
    st, info = Stats(), C.c_int(0)
    _check(lib().pdgstrf3d_b200(C.byref(view), C.byref(o), C.byref(st), C.byref(info)))
    del keep
    return info.value, st


def pzgstrf3d(prob, z=0, **opt):
    """pzgstrf3d_b200 (SRC/complex16/pzgstrf3d.c:120): factor layer z of a complex128 `prob` in place."""
    require_gpu()
    if not _is_complex(prob.dtype):
        raise TypeError("pzgstrf3d needs a complex128 problem")
    view, keep = make_view(prob, z)
    o = make_options(prob, **opt)
    st, info = Stats(), C.c_int(0)
    _check(lib().pzgstrf3d_b200(C.byref(view), C.byref(o), C.byref(st), C.byref(info)))
    del keep
    return info.value, st


# ---- kernel-level entry points -------------------------------------------------------------------
def k_diag_lu(a, replace_tiny=0, thresh=0.0, col0=0):
    require_gpu()
    z = _is_complex(np.asarray(a).dtype)
    a = np.array(a, np.complex128 if z else np.float64, order="F", copy=True)
    ns = a.shape[1]
    info, tiny = C.c_int(0), C.c_int(0)
    _check(_fn("k_diag_lu", z)(a.ctypes.data_as(C.c_void_p), ns, a.shape[0], replace_tiny, C.c_double(thresh),
                                    col0, C.byref(info), C.byref(tiny)))
    return a, info.value, tiny.value


def k_trsm(lu, x, ucase):
    require_gpu()
    z = _is_complex(np.asarray(lu).dtype) or _is_complex(np.asarray(x).dtype)
    dt = np.complex128 if z else np.float64
    lu = np.array(lu, dt, order="F", copy=True)
    x = np.array(x, dt, order="F", copy=True)
    ns = lu.shape[1]
    if ucase:
        _check(_fn("k_trsm_u", z)(lu.ctypes.data_as(C.c_void_p), lu.shape[0], ns, x.ctypes.data_as(C.c_void_p),
                                       x.shape[1], x.shape[0]))
    else:
        _check(_fn("k_trsm_l", z)(lu.ctypes.data_as(C.c_void_p), lu.shape[0], ns, x.ctypes.data_as(C.c_void_p),
                                       x.shape[0], x.shape[0]))
    return x


def k_gemm_sub(a, b, c, reps=0):
    require_gpu()
    z = any(_is_complex(np.asarray(t).dtype) for t in (a, b, c))
    dt = np.complex128 if z else np.float64
    a = np.array(a, dt, order="F", copy=True)
    b = np.array(b, dt, order="F", copy=True)
    c = np.array(c, dt, order="F", copy=True)
    m, k = a.shape
    n = b.shape[1]
    ms = C.c_float(0)
    _check(_fn("k_gemm_sub", z)(m, n, k, a.ctypes.data_as(C.c_void_p), a.shape[0], b.ctypes.data_as(C.c_void_p),
                                     b.shape[0], c.ctypes.data_as(C.c_void_p), c.shape[0], reps, C.byref(ms)))
    return c, ms.value
