"""oracle/selinv.py -- TEST INFRASTRUCTURE: a NumPy / SciPy restatement of the selected inversion of slu_b200_selinv.

On the panel layout of an LUProblem layer holding the factors F = L U (L panels nsupr x ns, U panels as skylines), it
computes H = F^-T at every stored position of L + U, supernode by supernode from the last to the first (every Schur
destination of supernode K lies in a supernode after K):

    M      = H(R, C)                          gathered from the panels of the later supernodes
    P_RK   = -M U_KC^T
    H(R,K) =  P_RK U_KK^-T
    H(K,C) = -L_KK^-T L_RK^T M
    H(K,K) =  L_KK^-T (I - L_RK^T P_RK) U_KK^-T  ( = L_KK^-T (U_KK^-T - L_RK^T H(R,K)) )

R = the sub-diagonal rows of L panel K, C = the packed columns of U panel K.  A^-1(i, j) = H(perm[j], perm[i]).
Every solve is a LAPACK substitution.  H(K,K) is solved from both sides, as slu_selinv.cu does: the explicit U_KK^-T of
the second form is not backward stable for L_KK^T H(K,K) U_KK^T = I - L_RK^T H(R,K) U_KK^T when U_KK is ill-conditioned
(pivots replaced by a threshold put it past its bound in tests/backward.py).  Only tests import this module."""
import numpy as np
import scipy.linalg as sla

from superlu_dist_b200.problem import BC_HEADER, BR_HEADER, LB_DESCRIPTOR, UB_DESCRIPTOR


class _Panels:
    """Index of one layer: per supernode its L rows, its packed U columns with their first rows and skyline offsets,
    and sorted lookup keys (supernode * n + row / column) into both."""

    def __init__(self, prob, layer):
        self.prob, self.layer = prob, layer
        n, xsup = prob.n, np.asarray(prob.xsup, np.int64)
        self.xsup = xsup
        self.supno = np.repeat(np.arange(prob.nsupers), np.diff(xsup))
        self.lrows, self.ucols, self.ufst, self.useg = {}, {}, {}, {}
        lk, lp, uk, uo = [], [], [], []
        for k in np.nonzero(layer.held)[0]:
            klst = int(xsup[k + 1])
            if prob.lidx_off[k + 1] > prob.lidx_off[k]:
                idx = prob.lidx[prob.lidx_off[k]:prob.lidx_off[k + 1]]
                w, rows = BC_HEADER, []
                for _ in range(int(idx[0])):
                    nb = int(idx[w + 1])
                    rows.append(idx[w + LB_DESCRIPTOR:w + LB_DESCRIPTOR + nb])
                    w += LB_DESCRIPTOR + nb
                rows = np.concatenate(rows).astype(np.int64)
                self.lrows[k] = rows
                lk.append(k * n + rows)
                lp.append(layer.lval_off[k] + np.arange(len(rows)))   # + column * nsupr at lookup
            cols, fsts = [], []
            if prob.uidx_off[k + 1] > prob.uidx_off[k]:
                idx = prob.uidx[prob.uidx_off[k]:prob.uidx_off[k + 1]]
                u = BR_HEADER
                for _ in range(int(idx[0])):
                    jb = int(idx[u])
                    jf, jns = int(xsup[jb]), int(xsup[jb + 1] - xsup[jb])
                    fst = idx[u + UB_DESCRIPTOR:u + UB_DESCRIPTOR + jns].astype(np.int64)
                    keep = fst < klst
                    cols.append(np.arange(jf, jf + jns)[keep])
                    fsts.append(fst[keep])
                    u += UB_DESCRIPTOR + jns
            cols = np.concatenate(cols) if cols else np.zeros(0, np.int64)
            fsts = np.concatenate(fsts) if fsts else np.zeros(0, np.int64)
            seg = np.concatenate([[0], np.cumsum(klst - fsts)])[:-1]
            self.ucols[k], self.ufst[k], self.useg[k] = cols, fsts, seg
            uk.append(k * n + cols)
            uo.append(layer.uval_off[k] + seg - fsts)                 # + row at lookup
        self.nsupr_of = np.zeros(prob.nsupers, np.int64)
        for k, rows in self.lrows.items():
            self.nsupr_of[k] = len(rows)
        cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)  # noqa: E731
        lk, lp, uk, uo = cat(lk), cat(lp), cat(uk), cat(uo)
        o = np.argsort(lk, kind="stable")
        self.lkey, self.lpos = lk[o], lp[o]
        o = np.argsort(uk, kind="stable")
        self.ukey, self.uoff = uk[o], uo[o]

    def lpanel(self, vals, k):
        """L panel k of an lval-shaped array as an nsupr x ns view"""
        ns, nsupr = int(self.xsup[k + 1] - self.xsup[k]), int(self.nsupr_of[k])
        o = int(self.layer.lval_off[k])
        return vals[o:o + ns * nsupr].reshape(ns, nsupr).T

    def upanel(self, vals, k):
        """U panel k of a uval-shaped array, dense-packed ns x ncols (zero above the skylines)"""
        f, klst = int(self.xsup[k]), int(self.xsup[k + 1])
        cols, fst, seg = self.ucols[k], self.ufst[k], self.useg[k]
        out = np.zeros((klst - f, len(cols)), vals.dtype)
        o = int(self.layer.uval_off[k])
        for j in range(len(cols)):
            out[fst[j] - f:, j] = vals[o + seg[j]:o + seg[j] + klst - fst[j]]
        return out

    def gather(self, hl, hu, rows, cols):
        """H(rows, cols) from the panels (every pair must be stored)"""
        n = self.prob.n
        ib, jb = self.supno[rows][:, None], self.supno[cols][None, :]
        inl = ib >= jb
        r2, c2 = np.broadcast_to(rows[:, None], inl.shape), np.broadcast_to(cols[None, :], inl.shape)
        out = np.empty(inl.shape, hl.dtype)
        # L panel of supno(col): row position of `row`, column col - xsup
        jj, rr, cc = np.broadcast_to(jb, inl.shape)[inl], r2[inl], c2[inl]
        q = np.searchsorted(self.lkey, jj * n + rr)
        assert (q < len(self.lkey)).all() and (self.lkey[np.minimum(q, len(self.lkey) - 1)] == jj * n + rr).all(), "L slot missing"
        out[inl] = hl[self.lpos[q] + (cc - self.xsup[jj]) * self.nsupr_of[jj]]
        # U panel of supno(row): skyline offset of column col, plus row
        ii, rr, cc = np.broadcast_to(ib, inl.shape)[~inl], r2[~inl], c2[~inl]
        q = np.searchsorted(self.ukey, ii * n + cc)
        assert (q < len(self.ukey)).all() and (self.ukey[np.minimum(q, len(self.ukey) - 1)] == ii * n + cc).all(), "U slot missing"
        out[~inl] = hu[self.uoff[q] + rr]
        return out


def selinv(prob, layer):
    """H = F^-T on every stored position of the factors in `layer` -> (hl, hu) shaped like layer.lval / layer.uval"""
    P = _Panels(prob, layer)
    hl = np.zeros_like(layer.lval)
    hu = np.zeros_like(layer.uval)
    held = np.nonzero(layer.held)[0]
    for k in held[::-1]:
        f, klst = int(P.xsup[k]), int(P.xsup[k + 1])
        ns = klst - f
        Lp = P.lpanel(layer.lval, k)
        Lkk = np.tril(Lp[:ns], -1) + np.eye(ns)
        Ukk = np.triu(Lp[:ns])
        Lrk = Lp[ns:]
        Ukc = P.upanel(layer.uval, k)
        R, C = P.lrows[k][ns:], P.ucols[k]
        M = P.gather(hl, hu, R, C) if len(R) and len(C) else np.zeros((len(R), len(C)), layer.lval.dtype)
        Prk = -(M @ Ukc.T)
        Hrk = sla.solve_triangular(Ukk, Prk.T, lower=False).T if len(R) else np.zeros((0, ns), Prk.dtype)
        Hkc = -sla.solve_triangular(Lkk, Lrk.T @ M, trans="T", lower=True, unit_diagonal=True)
        Y = sla.solve_triangular(Lkk, np.eye(ns) - Lrk.T @ Prk, trans="T", lower=True, unit_diagonal=True)
        Hkk = sla.solve_triangular(Ukk, Y.T, lower=False).T
        Hp = P.lpanel(hl, k)            # a view: writes land in hl
        Hp[:ns] = Hkk
        Hp[ns:] = Hrk
        o = int(layer.uval_off[k])
        for j in range(len(C)):
            fst, seg = int(P.ufst[k][j]), int(P.useg[k][j])
            hu[o + seg:o + seg + klst - fst] = Hkc[fst - f:, j]
    return hl, hu


def logdet(prob, layer):
    """(sign, log |det F|) from the pivots of the factors in `layer`, as numpy.linalg.slogdet"""
    xsup = np.asarray(prob.xsup, np.int64)
    logabs, sign = 0.0, 1.0
    for k in np.nonzero(layer.held)[0]:
        ns = int(xsup[k + 1] - xsup[k])
        nsupr = int(prob.lidx[prob.lidx_off[k] + 1])
        o = int(layer.lval_off[k])
        d = layer.lval[o:o + ns * nsupr].reshape(ns, nsupr)[np.arange(ns), np.arange(ns)]
        logabs += float(np.sum(np.log(np.abs(d))))
        sign *= float(np.prod(np.sign(d)))
    return sign, logabs
