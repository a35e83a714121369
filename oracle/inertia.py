"""oracle/inertia.py -- TEST INFRASTRUCTURE: a NumPy restatement of slu_b200_inertia.

F = P A P^T = L U is factored with a symmetric permutation, no row exchanges and a unit-diagonal L.  For a real symmetric
(complex Hermitian) A, U = D L^T (D L^H), so by Sylvester's law the signs of the pivots u_ii (the diagonals of the
diagonal blocks of the L panels) are those of A's eigenvalues.  Only tests import this module."""
import numpy as np


def pivots(prob, layer):
    """The pivots u_ii of the factors in `layer`, supernode by supernode"""
    xsup = np.asarray(prob.xsup, np.int64)
    out = []
    for k in np.nonzero(layer.held)[0]:
        ns = int(xsup[k + 1] - xsup[k])
        nsupr = int(prob.lidx[prob.lidx_off[k] + 1])
        o = int(layer.lval_off[k])
        out.append(layer.lval[o:o + ns * nsupr].reshape(ns, nsupr)[np.arange(ns), np.arange(ns)])
    return np.concatenate(out) if out else np.zeros(0, layer.lval.dtype)


def inertia(prob, layer, thresh=None):
    """(neg, pos, tiny, defect) as slu_b200_inertia returns them: the pivots with Re u_ii < 0, the others, those with
    |u_ii| <= thresh (default prob.thresh), and max |Im u_ii| / |u_ii| (0.0 for real factors)"""
    d = pivots(prob, layer)
    thresh = prob.thresh if thresh is None else thresh
    a = np.abs(d)
    neg = int(np.count_nonzero(d.real < 0))
    defect = float(np.max(np.abs(d.imag)[a > 0] / a[a > 0], initial=0.0)) if np.iscomplexobj(d) else 0.0
    return neg, len(d) - neg, int(np.count_nonzero(a <= thresh)), defect
