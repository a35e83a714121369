"""LUProblem: the input/output of `pdgstrf3d` held exactly as the reference holds it.

Structure (identical on every rank): ``xsup`` (Glu_persist_t), the L block-column and U block-row
index arrays in the layout of SRC/include/superlu_defs.h:156-204, the supernodal etree and the
Z-forest partition of dtrf3Dpartition_t (superlu_ddefs.h:317-337).  Values: one ``Layer`` per Z
coordinate holding the Lnzval/Unzval arrays of the supernodes that layer owns (dLocalLU_t).

Only 1 x 1 x Pz process grids are modelled here (nprow = npcol = 1): local block index == global
supernode index.
"""
import ctypes as C

import numpy as np

from . import hostlib

BC_HEADER, LB_DESCRIPTOR, BR_HEADER, UB_DESCRIPTOR = 2, 2, 3, 2


def my_tree_idxs(npdep, z):
    """getGridTrees (SRC/prec-independent/supernodal_etree.c:840-851)."""
    max_lvl = int(np.log2(npdep)) + 1
    idx = [npdep - 1 + z]
    for _ in range(1, max_lvl):
        idx.append((idx[-1] - 1) // 2)
    return np.array(idx, np.int32)


def my_zero_tr_idxs(npdep, z):
    """getReplicatedTrees (supernodal_etree.c:853-871)."""
    max_lvl = int(np.log2(npdep)) + 1
    return np.array([1 if z % (1 << i) else 0 for i in range(max_lvl)], np.int32)


class Layer:
    """Value arrays of one Z-layer (offsets are zero-length for supernodes the layer does not hold)."""

    def __init__(self, z, held, lval_off, uval_off, lval, uval, keep=None):
        self.z = z
        self.held = held            # bool [nsupers]
        self.lval_off = lval_off    # int64 [nsupers+1]
        self.uval_off = uval_off
        self.lval = lval            # float64 arena
        self.uval = uval
        self._keep = keep           # owner of pinned memory, if any

    def copy(self):
        return Layer(self.z, self.held, self.lval_off, self.uval_off, self.lval.copy(), self.uval.copy())


class LUProblem:
    def __init__(self):
        self.n = 0
        self.nsupers = 0
        self.xsup = None
        self.setree = None
        self.lidx_off = self.lidx = self.uidx_off = self.uidx = None
        self.lval_len = None        # int64 [nsupers]  doubles in L panel k
        self.uval_len = None        # int64 [nsupers]  doubles in U panel k (skyline)
        self.npdep = 1
        self.max_lvl = 1
        self.forest_of = None       # int32 [nsupers], heap numbering
        self.forest_nodes = None    # list of int32 arrays
        self.perm = None
        self.ops_fact = None        # reference-accounting flops, when known analytically
        self.ops_schur = None
        self.replace_tiny_pivot = 0
        self.thresh = 0.0
        self.dtype = np.dtype(np.float64)   # complex128 for the doublecomplex mirror (pzgstrf3d)
        self.nschur = 0                     # the last nschur unknowns form whole supernodes (from_matrix(..., nschur))
        self.layers = {}

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_symbolic(cls, sym, npdep=1):
        p = cls()
        p.n, p.nsupers = sym.n, sym.nsupers
        p.xsup, p.setree, p.perm = sym.xsup, sym.setree, sym.perm
        p.lidx_off, p.lidx, p.uidx_off, p.uidx = sym.lidx_off, sym.lidx, sym.uidx_off, sym.uidx
        p.lval_len = np.diff(sym.lval_off)
        p.uval_len = np.diff(sym.uval_off)
        p.ops_fact, p.ops_schur = sym.ops_fact, sym.ops_schur
        p.set_grid(npdep)
        return p

    @classmethod
    def from_matrix(cls, rowptr, colind, val, perm=None, relax=32, maxsup=256, npdep=1, layers=(0,),
                    alloc=None, amalg=0.05, nschur=0):
        """nschur > 0: the unknowns perm sends to n - nschur .. n - 1 stay last and form whole supernodes (the layout of
        capi.SchurHandle; hostlib.schur_order makes such a perm)."""
        n = len(rowptr) - 1
        sym = hostlib.Symbolic(n, rowptr, colind, perm, relax, maxsup, amalg, nschur)
        p = cls.from_symbolic(sym, npdep)
        p.nschur = int(nschur)
        for z in layers:
            p.add_layer(z, alloc=alloc)
            p.fill_layer(z, rowptr, colind, val)
        return p

    @classmethod
    def from_dump(cls, pre):
        """Build from the records of a `.pre` dump of the reference (dumpio.read_records)."""
        p = cls()
        p.n, p.nsupers = int(pre["n"][0]), int(pre["nsupers"][0])
        if int(pre["nprow"][0]) != 1 or int(pre["npcol"][0]) != 1:
            raise ValueError("only 1 x 1 x Pz dumps are supported")
        ns = p.nsupers
        p.xsup = pre["xsup"].astype(np.int32)
        p.setree = pre["setree"].astype(np.int32)
        p.replace_tiny_pivot = int(pre["ReplaceTinyPivot"][0])
        if any(k.startswith("Lval:") and np.iscomplexobj(a) for k, a in pre.items()):
            p.dtype = np.dtype(np.complex128)
        p.thresh = float(pre["thresh"][0])
        empty_i = np.zeros(0, np.int32)
        li = [pre.get(f"Lidx:{k}", empty_i) for k in range(ns)]
        ui = [pre.get(f"Uidx:{k}", empty_i) for k in range(ns)]
        p.lidx_off = np.concatenate([[0], np.cumsum([len(a) for a in li])]).astype(np.int64)
        p.uidx_off = np.concatenate([[0], np.cumsum([len(a) for a in ui])]).astype(np.int64)
        p.lidx = np.concatenate(li + [empty_i]).astype(np.int32)
        p.uidx = np.concatenate(ui + [empty_i]).astype(np.int32)
        if len(p.lidx) == 0:
            p.lidx = np.zeros(1, np.int32)
        if len(p.uidx) == 0:
            p.uidx = np.zeros(1, np.int32)
        sizes = np.diff(p.xsup).astype(np.int64)
        p.lval_len = np.array([int(a[1]) * int(sizes[k]) if len(a) else 0 for k, a in enumerate(li)], np.int64)
        p.uval_len = np.array([int(a[1]) if len(a) else 0 for a in ui], np.int64)
        p.npdep = int(pre["npdep"][0])
        p.max_lvl = int(pre["maxLvl"][0])
        nf = (1 << p.max_lvl) - 1
        p.forest_nodes = [pre[f"forest_nodes:{f}"].astype(np.int32) for f in range(nf)]
        p.forest_of = np.full(ns, -1, np.int32)
        for f, nodes in enumerate(p.forest_nodes):
            p.forest_of[nodes] = f
        z = int(pre["mydep"][0])
        lay = p.add_layer(z)
        p.load_values(lay, pre)
        return p

    def prune_u(self, rowptr, colind):
        """Cut every U block row down to the exact skyline of the unsymmetric F = P A P^T (A: the CSR pattern of the
        matrix this problem was built from, perm[old] = new), as the reference stores unsymmetric patterns: per column j
        of U panel k only the segment [fstnz, klst), columns with an empty segment and blocks without columns dropped.
        L keeps the structure of P (A + A^T) P^T, a valid superset.  Call before any layer exists.

        fstnz_k(j) is the first row of k with F(i, j) != 0, or the first row of k that an earlier supernode s updates
        in column j: s's pruned U panel has column j and s's L panel lists rows of k.  The diagonal block of k is dense,
        so below fstnz every row of the column may be non-zero.  The analytic operation counts no longer apply."""
        if self.layers:
            raise ValueError("prune_u changes the U layout: call it before add_layer")
        n, ns_all = self.n, self.nsupers
        xsup = np.asarray(self.xsup, np.int64)
        supno = np.repeat(np.arange(ns_all), np.diff(xsup))
        # the U column list of every panel (keys k * n + j, ascending) and each block's extent in it
        keys, first = [], np.zeros(ns_all + 1, np.int64)
        blocks = [None] * ns_all
        for k in range(ns_all):
            cols = []
            if self.uidx_off[k + 1] > self.uidx_off[k]:
                idx = self.uidx[self.uidx_off[k]:self.uidx_off[k + 1]]
                klst, u, blk = int(xsup[k + 1]), BR_HEADER, []
                for _ in range(int(idx[0])):
                    jb = int(idx[u])
                    jf, jns = int(xsup[jb]), int(xsup[jb + 1] - xsup[jb])
                    c = np.nonzero(idx[u + UB_DESCRIPTOR:u + UB_DESCRIPTOR + jns] < klst)[0] + jf
                    blk.append(jb)
                    cols.append(c)
                    u += UB_DESCRIPTOR + jns
                blocks[k] = blk
            cols = np.concatenate(cols) if cols else np.zeros(0, np.int64)
            keys.append(k * n + cols)
            first[k + 1] = first[k] + len(cols)
        keys = np.concatenate(keys) if keys else np.zeros(0, np.int64)
        fst = np.repeat(xsup[1:], np.diff(first))              # klst: empty

        def lookup(k, cols):
            q = np.searchsorted(keys, k * n + cols)
            if np.any(q >= len(keys)) or np.any(keys[np.minimum(q, len(keys) - 1)] != k * n + cols):
                raise ValueError("F has an entry outside the U structure of P (A + A^T) P^T")
            return q
        # entries of F above the diagonal blocks
        rowptr, colind = np.asarray(rowptr), np.asarray(colind)
        perm = np.asarray(self.perm, np.int64)
        fi = perm[np.repeat(np.arange(n), np.diff(rowptr))]
        fj = perm[colind]
        up = supno[fi] < supno[fj]
        fi, fj = fi[up], fj[up]
        np.minimum.at(fst, lookup(supno[fi], fj), fi)
        # updates of earlier supernodes, in ascending order (fstnz of s is final once every s' < s has been applied)
        for s in range(ns_all):
            if first[s + 1] == first[s]:
                continue
            live = fst[first[s]:first[s + 1]] < xsup[s + 1]
            cols_s = keys[first[s]:first[s + 1]][live] - s * n
            if not len(cols_s):
                continue
            idx = self.lidx[self.lidx_off[s]:self.lidx_off[s + 1]]
            w = BC_HEADER
            for b in range(int(idx[0])):
                ib, nb = int(idx[w]), int(idx[w + 1])
                if b:
                    tgt = cols_s[cols_s >= xsup[ib + 1]]
                    if len(tgt):
                        q = lookup(ib, tgt)
                        fst[q] = np.minimum(fst[q], int(idx[w + LB_DESCRIPTOR]))
                w += LB_DESCRIPTOR + nb
        # the new U index arrays
        out, off, vlen = [], [0], np.zeros(ns_all, np.int64)
        for k in range(ns_all):
            if blocks[k] is None:
                off.append(off[-1])
                continue
            klst = int(xsup[k + 1])
            colfst = dict(zip((keys[first[k]:first[k + 1]] - k * n).tolist(), fst[first[k]:first[k + 1]].tolist()))
            body, nblk, nnz = [], 0, 0
            for jb in blocks[k]:
                jf, jns = int(xsup[jb]), int(xsup[jb + 1] - xsup[jb])
                f = [colfst.get(jf + c, klst) for c in range(jns)]
                bnnz = sum(klst - x for x in f)
                if bnnz:
                    body += [jb, bnnz] + f
                    nblk += 1
                    nnz += bnnz
            if nblk:
                out.append(np.array([nblk, nnz, BR_HEADER + len(body)] + body, np.int32))
                off.append(off[-1] + BR_HEADER + len(body))
                vlen[k] = nnz
            else:
                off.append(off[-1])
        self.uidx = np.concatenate(out) if out else np.zeros(1, np.int32)
        self.uidx_off = np.array(off, np.int64)
        self.uval_len = vlen
        self.ops_fact = self.ops_schur = None
        return self

    def load_values(self, layer, rec):
        for k in range(self.nsupers):
            a = rec.get(f"Lval:{k}")
            if a is not None:
                layer.lval[layer.lval_off[k]:layer.lval_off[k + 1]] = a
            a = rec.get(f"Uval:{k}")
            if a is not None:
                layer.uval[layer.uval_off[k]:layer.uval_off[k + 1]] = a

    # ------------------------------------------------------------------ grid / forests
    def set_grid(self, npdep):
        if npdep & (npdep - 1):
            raise ValueError("npdep must be a power of two (EXAMPLE/pddrive3d.c:132)")
        self.npdep = npdep
        self.max_lvl = int(np.log2(npdep)) + 1
        sizes = np.diff(self.xsup).astype(np.float64)
        nrows = np.array([self.lidx[self.lidx_off[k] + 1] for k in range(self.nsupers)], np.float64) \
            if self.nsupers < 200000 else self._nrows_vec()
        weight = sizes * nrows * nrows
        self.forest_of = hostlib.forests(self.setree, weight, self.max_lvl)
        nf = (1 << self.max_lvl) - 1
        order = np.argsort(self.forest_of, kind="stable").astype(np.int32)
        counts = np.bincount(self.forest_of, minlength=nf)
        starts = np.concatenate([[0], np.cumsum(counts)])
        self.forest_nodes = [order[starts[f]:starts[f + 1]].copy() for f in range(nf)]

    def _nrows_vec(self):
        return self.lidx[self.lidx_off[:-1] + 1].astype(np.float64)

    def held_mask(self, z):
        held = np.zeros(self.nsupers, bool)
        for f in my_tree_idxs(self.npdep, z):
            held[self.forest_nodes[f]] = True
        return held

    def add_layer(self, z, alloc=None):
        """Allocate the value arenas of Z-layer z (alloc(nbytes) -> (address, keepalive) for pinned memory)."""
        held = self.held_mask(z)
        lval_off = np.concatenate([[0], np.cumsum(np.where(held, self.lval_len, 0))]).astype(np.int64)
        uval_off = np.concatenate([[0], np.cumsum(np.where(held, self.uval_len, 0))]).astype(np.int64)
        nl, nu = int(lval_off[-1]), int(uval_off[-1])
        keep = None
        if alloc is None:
            lval = np.zeros(max(nl, 1), self.dtype)
            uval = np.zeros(max(nu, 1), self.dtype)
        else:
            if self.dtype != np.float64:
                raise ValueError("pinned allocation is wired for float64 only")
            a1, k1 = alloc(8 * max(nl, 1))
            a2, k2 = alloc(8 * max(nu, 1))
            lval = np.ctypeslib.as_array((C.c_double * max(nl, 1)).from_address(a1))
            uval = np.ctypeslib.as_array((C.c_double * max(nu, 1)).from_address(a2))
            keep = (k1, k2)
        lay = Layer(z, held, lval_off, uval_off, lval, uval, keep)
        self.layers[z] = lay
        return lay

    def fill_layer(self, z, rowptr, colind, val):
        """pddistribute3d + dinit3DLUstructForest: A into the panels; replicated ancestors start at 0.  float64 only: the
        host fill writes doubles, so a complex matrix goes into float64 arenas part by part (real, then imaginary) and the
        two results are combined."""
        lay = self.layers[z]
        if np.iscomplexobj(val) or np.iscomplexobj(lay.lval) or np.iscomplexobj(lay.uval):
            raise TypeError("LUProblem.fill_layer fills float64 layers with float64 values; fill a complex matrix part by "
                            "part (real, then imaginary part into float64 arenas) and combine the two")
        active = np.zeros(self.nsupers, np.int8)
        trees, zero = my_tree_idxs(self.npdep, z), my_zero_tr_idxs(self.npdep, z)
        for f, zr in zip(trees, zero):
            if not zr:
                active[self.forest_nodes[f]] = 1
        hostlib.lib().sluh_fill_values(
            self.n, np.ascontiguousarray(rowptr, np.int32), np.ascontiguousarray(colind, np.int32),
            np.ascontiguousarray(val, np.float64), self.perm, self.nsupers, self.xsup, self.lidx_off,
            self.lidx, lay.lval_off, lay.lval.ctypes.data_as(C.c_void_p), self.uidx_off, self.uidx,
            lay.uval_off, lay.uval.ctypes.data_as(C.c_void_p), active.ctypes.data_as(C.c_void_p))

    # ------------------------------------------------------------------ raw pointer tables
    def pointer_tables(self, layer):
        """Arrays of per-block pointers (NULL where the layer holds nothing), as dLocalLU_t has them."""
        li = np.where(layer.held & (np.diff(self.lidx_off) > 0),
                      self.lidx.ctypes.data + 4 * self.lidx_off[:-1], 0).astype(np.uint64)
        lv = np.where(layer.held & (self.lval_len > 0),
                      layer.lval.ctypes.data + layer.lval.itemsize * layer.lval_off[:-1], 0).astype(np.uint64)
        ui = np.where(layer.held & (np.diff(self.uidx_off) > 0),
                      self.uidx.ctypes.data + 4 * self.uidx_off[:-1], 0).astype(np.uint64)
        uv = np.where(layer.held & (self.uval_len > 0),
                      layer.uval.ctypes.data + layer.uval.itemsize * layer.uval_off[:-1], 0).astype(np.uint64)
        # a U panel with an index but zero values still needs a non-NULL value pointer
        uv = np.where((ui != 0) & (uv == 0), layer.uval.ctypes.data, uv).astype(np.uint64)
        return li, lv, ui, uv

    # ------------------------------------------------------------------ checker
    def matvec(self, layers, x, mode):
        """y = M x with M assembled from the given layers (each supernode taken from the first layer
        in `layers` that is listed as its owner by `owner_of`); mode 0 plain, 1 factors."""
        x = np.ascontiguousarray(x, np.float64)
        nvec = 1 if x.ndim == 1 else x.shape[0]
        li = np.zeros(self.nsupers, np.uint64)
        lv = np.zeros(self.nsupers, np.uint64)
        ui = np.zeros(self.nsupers, np.uint64)
        uv = np.zeros(self.nsupers, np.uint64)
        for lay, sel in layers:
            a, b, c, d = self.pointer_tables(lay)
            m = sel & lay.held
            li[m], lv[m], ui[m], uv[m] = a[m], b[m], c[m], d[m]
        y = np.zeros_like(x)
        hostlib.lib().sluh_panel_matvec(mode, self.n, self.nsupers, self.xsup,
                                        li.ctypes.data_as(C.c_void_p), lv.ctypes.data_as(C.c_void_p),
                                        ui.ctypes.data_as(C.c_void_p), uv.ctypes.data_as(C.c_void_p),
                                        nvec, x.reshape(-1), y.reshape(-1))
        return y

    def final_owner_masks(self):
        """After pdgstrf3d each supernode's factors live on the layer that factored it
        (SURVEY 8b): forest f at Z-tree level lvl is factored by the layer with z % 2^lvl == 0."""
        masks = {}
        for z in range(self.npdep):
            m = np.zeros(self.nsupers, bool)
            for f, zr in zip(my_tree_idxs(self.npdep, z), my_zero_tr_idxs(self.npdep, z)):
                if not zr:
                    m[self.forest_nodes[f]] = True
            masks[z] = m
        return masks

    # ------------------------------------------------------------------ dense views (small tests)
    def dense(self, layer, factored):
        """(A) or (L, U) as dense arrays assembled from one layer's panels (small n only)."""
        n = self.n
        L = np.zeros((n, n), self.dtype)
        U = np.zeros((n, n), self.dtype)
        for k in range(self.nsupers):
            if not layer.held[k]:
                continue
            f, ns = int(self.xsup[k]), int(self.xsup[k + 1] - self.xsup[k])
            klst = f + ns
            if self.lidx_off[k + 1] > self.lidx_off[k]:
                idx = self.lidx[self.lidx_off[k]:self.lidx_off[k + 1]]
                nsupr = int(idx[1])
                vals = layer.lval[layer.lval_off[k]:layer.lval_off[k + 1]].reshape(ns, nsupr).T
                w, rows = BC_HEADER, []
                for _ in range(int(idx[0])):
                    nb = int(idx[w + 1])
                    rows.extend(idx[w + 2:w + 2 + nb])
                    w += LB_DESCRIPTOR + nb
                rows = np.array(rows)
                if factored:
                    for i, r in enumerate(rows):
                        for c in range(ns):
                            if r > f + c:
                                L[r, f + c] = vals[i, c]
                            else:
                                U[r, f + c] = vals[i, c]
                else:
                    L[rows[:, None], np.arange(f, klst)[None, :]] = vals
            if self.uidx_off[k + 1] > self.uidx_off[k]:
                idx = self.uidx[self.uidx_off[k]:self.uidx_off[k + 1]]
                uv = layer.uval[layer.uval_off[k]:layer.uval_off[k + 1]]
                u, seg = BR_HEADER, 0
                for _ in range(int(idx[0])):
                    jb = int(idx[u])
                    jf, jns = int(self.xsup[jb]), int(self.xsup[jb + 1] - self.xsup[jb])
                    for c in range(jns):
                        fst = int(idx[u + UB_DESCRIPTOR + c])
                        if fst < klst:
                            (U if factored else L)[fst:klst, jf + c] = uv[seg:seg + klst - fst]
                            seg += klst - fst
                    u += UB_DESCRIPTOR + jns
        if factored:
            return L + np.eye(n), U
        return L


class Local2D:
    """The pieces of one Z-layer that process (myrow, mycol) of a Pr x Pc grid holds, exactly as
    pddistribute3d leaves them (SRC/include/superlu_defs.h:270-279): block (I, J) lives on process
    (I mod Pr, J mod Pc); L block column J is the local panel J / Pc of process column J mod Pc and lists
    only the row blocks I with I mod Pr == myrow; U block row I is the local panel I / Pr of process row
    I mod Pr and lists only the column blocks J with J mod Pc == mycol."""

    def __init__(self, prob, layer, nprow, npcol, myrow, mycol):
        self.prob, self.layer = prob, layer
        self.nprow, self.npcol, self.myrow, self.mycol = nprow, npcol, myrow, mycol
        ns_all = prob.nsupers
        self.nbc, self.nbr = -(-ns_all // npcol), -(-ns_all // nprow)
        self.lidx, self.lval = [None] * self.nbc, [None] * self.nbc
        self.uidx, self.uval = [None] * self.nbr, [None] * self.nbr
        self._lmap, self._umap = {}, {}     # k -> positions of my entries inside the full panel arrays
        xsup = prob.xsup
        for k in np.nonzero(layer.held)[0]:
            ns = int(xsup[k + 1] - xsup[k])
            if k % npcol == mycol and prob.lidx_off[k + 1] > prob.lidx_off[k]:
                idx = prob.lidx[prob.lidx_off[k]:prob.lidx_off[k + 1]]
                nsupr, w, row0, out, rowsel = int(idx[1]), BC_HEADER, 0, [], []
                for _ in range(int(idx[0])):
                    ib, nb = int(idx[w]), int(idx[w + 1])
                    if ib % nprow == myrow:
                        out.append(idx[w:w + LB_DESCRIPTOR + nb])
                        rowsel.append(np.arange(row0, row0 + nb))
                    row0 += nb
                    w += LB_DESCRIPTOR + nb
                if out:
                    rowsel = np.concatenate(rowsel)
                    li = np.concatenate([[len(out), len(rowsel)]] + out).astype(np.int32)
                    pos = (rowsel[None, :] + nsupr * np.arange(ns)[:, None]).reshape(-1)   # column-major gather
                    self.lidx[k // npcol] = li
                    self.lval[k // npcol] = np.ascontiguousarray(layer.lval[layer.lval_off[k] + pos])
                    self._lmap[k] = pos
            if k % nprow == myrow and prob.uidx_off[k + 1] > prob.uidx_off[k]:
                idx = prob.uidx[prob.uidx_off[k]:prob.uidx_off[k + 1]]
                klst, u, seg, out, sel, nnz = int(xsup[k + 1]), BR_HEADER, 0, [], [], 0
                for _ in range(int(idx[0])):
                    jb = int(idx[u])
                    jns = int(xsup[jb + 1] - xsup[jb])
                    blk_nnz = int(np.sum(klst - idx[u + UB_DESCRIPTOR:u + UB_DESCRIPTOR + jns]))
                    if jb % npcol == mycol:
                        out.append(idx[u:u + UB_DESCRIPTOR + jns])
                        sel.append(np.arange(seg, seg + blk_nnz))
                        nnz += blk_nnz
                    seg += blk_nnz
                    u += UB_DESCRIPTOR + jns
                if out:
                    body = np.concatenate(out)
                    ui = np.concatenate([[len(out), nnz, BR_HEADER + len(body)], body]).astype(np.int32)
                    pos = np.concatenate(sel) if nnz else np.zeros(0, np.int64)
                    self.uidx[k // nprow] = ui
                    self.uval[k // nprow] = np.ascontiguousarray(layer.uval[layer.uval_off[k] + pos]) if nnz else np.zeros(1, layer.uval.dtype)
                    self._umap[k] = pos

    def pointer_tables(self):
        def tab(arrs):
            return np.array([a.ctypes.data if a is not None else 0 for a in arrs], np.uint64)
        return tab(self.lidx), tab(self.lval), tab(self.uidx), tab(self.uval)

    def scatter_back(self, out_layer):
        """Write my (factored) pieces into a full-layout Layer (for checking against the oracle)."""
        for k, pos in self._lmap.items():
            out_layer.lval[out_layer.lval_off[k] + pos] = self.lval[k // self.npcol]
        for k, pos in self._umap.items():
            if len(pos):
                out_layer.uval[out_layer.uval_off[k] + pos] = self.uval[k // self.nprow]

    def owned_positions(self):
        """(L positions, U positions) in the full layer arenas of the entries I hold."""
        lay = self.layer
        lp = [lay.lval_off[k] + pos for k, pos in self._lmap.items()]
        up = [lay.uval_off[k] + pos for k, pos in self._umap.items() if len(pos)]
        cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)  # noqa: E731
        return cat(lp), cat(up)
