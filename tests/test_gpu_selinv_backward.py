"""Selected inversion step by step on the GPU (test_selinv_backward_cpu.py shows the references meeting every bound on
these inputs, and the plain product with the explicit 16 x 16 inverses failing it): Handle.selinv in double and
doublecomplex, BatchHandle.selinv with B = 3 and a fill_csr_scaled handle with pivots replaced mid-block.  The GPU's own
factors are downloaded and H is read on every stored position through inv_entries.  A route passes when every step of
every supernode is within its bound (backward.selinv_ratios) and within 16 x max(the references' ratio on the same
factors, 8 u), the references being oracle/selinv.py (substitution) and backward.selinv_blocked with the correction
step.  logdet and inertia on the same handles must agree with the values from the downloaded pivots."""
import numpy as np
import pytest

import backward as bw
from oracle import inertia, selinv
from superlu_dist_b200 import capi
from test_gpu_selinv import csr_of, stored_positions
from test_gpu_trsm_consistent import REPLACE_DELTA, REPLACE_THRESH, make
from test_selinv_backward_cpu import INPUTS, unfactored

pytestmark = pytest.mark.gpu


def read_h(inv_entries, prob, lay):
    """H on every stored position through inv_entries (identity permutation: A^-1(i, j) = H(j, i)) -> (hl, hu) shaped
    like lay.lval / lay.uval, or stacks of them for a batched handle"""
    rows, cols, u = stored_positions(prob, lay)
    rp, ci, order = csr_of(cols, rows, prob.n)
    got = inv_entries(rp, ci, np.arange(prob.n, dtype=np.int32))
    vals = np.empty_like(got)
    vals[..., order] = got
    nl = len(lay.lval)
    hu = np.zeros(vals.shape[:-1] + lay.uval.shape, vals.dtype)
    hu[..., u] = vals[..., nl:]
    return vals[..., :nl], hu


def check(prob, hl, hu, label):
    """H from the GPU against the bounds and against the references on the factors in layer 0"""
    lay = prob.layers[0]
    scaled, raw = bw.selinv_ratios(prob, lay, hl, hu)
    base = np.maximum(bw.selinv_ratios(prob, lay, *selinv.selinv(prob, lay))[1],
                      bw.selinv_ratios(prob, lay, *bw.selinv_blocked(prob, lay, 1))[1])
    report = {s: (f"{q:.3g} of the bound", f"{r / bw.U:.3g} u", f"reference {b / bw.U:.3g} u")
              for s, q, r, b in zip(bw.SELINV_STEPS, scaled, raw, base)}
    assert (scaled <= 1).all() and (raw <= 16 * np.maximum(base, 8 * bw.U)).all(), (label, report)


def check_logdet_inertia(prob, got_logdet, got_inertia, thresh):
    lay = prob.layers[0]
    sign, la, tol, ptol = bw.pivot_logdet(prob, lay)
    gs, gl = got_logdet
    assert abs(gl - la) <= tol, (gl, la, tol)
    if np.iscomplexobj(lay.lval):
        assert abs(gs - sign) <= ptol, (gs, sign, ptol)
    else:
        assert gs == sign, (gs, sign)
    neg, pos, tiny, defect = inertia.inertia(prob, lay, thresh)
    assert tuple(got_inertia[:3]) == (neg, pos, tiny), (got_inertia, (neg, pos, tiny))
    assert abs(got_inertia[3] - defect) <= 4 * bw.U * defect, (got_inertia[3], defect)


@pytest.mark.parametrize("name", INPUTS)
def test_handle_selinv(name):
    prob = unfactored(name)
    h = capi.Handle(prob, 0)
    try:
        h.upload()
        assert h.factor() == 0
        h.selinv()
        h.download()
        check(prob, *read_h(h.inv_entries, prob, prob.layers[0]), name)
        check_logdet_inertia(prob, h.logdet(), h.inertia(), prob.thresh)
    finally:
        h.close()


@pytest.mark.parametrize("name", list(bw.PLANTED) + list(bw.ZPLANTED))
def test_batch_selinv(name):
    """B = 3 on one pattern: the planted factors, the same without small pivots, another planting"""
    cases = [make(name), make(name, 1, 1.0, 1.0), make(name, 2)]
    prob = cases[0][0]
    rp, ci = cases[0][2][:2]
    assert all(np.array_equal(c[2][1], ci) for c in cases)
    h = capi.BatchHandle(prob, 3)
    try:
        h.fill_csr(rp, ci, np.stack([c[2][2] for c in cases]), prob.perm)
        assert not h.factor().any()
        h.selinv()
        hl, hu = read_h(h.inv_entries, prob, prob.layers[0])
        sg, la = h.logdet()
        inr = h.inertia()
        for j in range(3):
            h.download(j)
            check(prob, hl[j], hu[j], (name, j))
            check_logdet_inertia(prob, (sg[j], la[j]), [x[j] for x in inr], prob.thresh)
    finally:
        h.close()


def test_fill_csr_scaled_replaced_pivots_mid_block():
    """The planted pivots of fem6 at 1e-10 replaced under a threshold of 1e-8, at in-block offsets 1, 7 and 14"""
    prob, _, (rp, ci, vals) = make("fem6", 0, REPLACE_DELTA)
    prob.replace_tiny_pivot, prob.thresh = 1, REPLACE_THRESH
    h = capi.Handle(prob, 0)
    try:
        h.fill_csr_scaled(rp, ci, vals, prob.perm, equil=False)
        assert h.factor() == 0
        assert h.stats().tiny_pivots > 0
        h.selinv()
        h.download()
        d = np.abs(bw.factors(prob, prob.layers[0])[1].diagonal())
        xsup = np.asarray(prob.xsup)
        off = (np.arange(prob.n) - xsup[np.searchsorted(xsup, np.arange(prob.n), side="right") - 1]) % 16
        assert set(off[d == REPLACE_THRESH]) & {1, 7, 14}
        check(prob, *read_h(h.inv_entries, prob, prob.layers[0]), "fem6 replaced")
        check_logdet_inertia(prob, h.logdet(), h.inertia(), REPLACE_THRESH)
    finally:
        h.close()
