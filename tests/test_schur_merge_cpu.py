"""Deferred Schur updates along supernode chains (options.reserved[6], DESIGN 4a), without a device: the nesting rule
restated in NumPy from the reference index arrays (lidx / uidx) must give the plan's count of deferred children and of
destination updates at every depth, and the flop counts must not move."""
import numpy as np
import pytest

from superlu_dist_b200 import capi
from util import poisson_problem

BIG = 96   # narrowest update (rows and columns) on the big-tile kernel


def _structure(prob):
    """Per supernode: the sub-diagonal L rows and the packed U columns, in stored order."""
    xsup = np.asarray(prob.xsup)
    rows, cols = [], []
    for k in range(prob.nsupers):
        ns = xsup[k + 1] - xsup[k]
        li = prob.lidx[prob.lidx_off[k]:prob.lidx_off[k + 1]]
        r, w = [], 2
        for _ in range(li[0]):
            nb = li[w + 1]
            r.extend(li[w + 2:w + 2 + nb])
            w += 2 + nb
        rows.append(np.asarray(r[ns:], np.int64))
        c = []
        if prob.uidx_off[k + 1] > prob.uidx_off[k]:
            ui = prob.uidx[prob.uidx_off[k]:prob.uidx_off[k + 1]]
            u = 3
            for _ in range(ui[0]):
                jb = ui[u]
                jns = xsup[jb + 1] - xsup[jb]
                fst = ui[u + 2:u + 2 + jns]
                c.extend(xsup[jb] + np.nonzero(fst < xsup[k + 1])[0])
                u += 2 + jns
        cols.append(np.asarray(c, np.int64))
    return xsup, rows, cols


def _merge(prob, depth):
    """-> (deferred children, REDs at depth 1, REDs at `depth`): a child k defers into parent p when k's rows and columns
    are p's columns followed by p's rows / columns, both updates are big, and p's GEMM stays within `depth` panels."""
    xsup, rows, cols = _structure(prob)
    supno = np.repeat(np.arange(prob.nsupers), np.diff(xsup))
    first = prob.n - prob.nschur if prob.nschur else prob.n
    panels = np.ones(prob.nsupers, np.int64)
    deferred, reds, saved = 0, 0, 0
    for k in range(prob.nsupers):
        m, n = len(rows[k]), len(cols[k])
        if xsup[k] >= first or m == 0 or n == 0:
            continue
        reds += m * n
        if depth < 2 or m < BIG or n < BIG:
            continue
        p = supno[rows[k][0]]
        mp, npc = len(rows[p]), len(cols[p])
        if xsup[p] >= first or mp < BIG or npc < BIG or panels[k] + panels[p] > depth:
            continue
        own = np.arange(xsup[p], xsup[p + 1])
        if np.array_equal(rows[k], np.concatenate([own, rows[p]])) and np.array_equal(cols[k], np.concatenate([own, cols[p]])):
            panels[p] += panels[k]
            deferred += 1
            saved += mp * npc
    return deferred, reds, reds - saved


CASES = [dict(N=20, leaf=8, relax=8, maxsup=64), dict(N=20, leaf=8, relax=37, maxsup=100),
         dict(N=24, leaf=16, relax=32, maxsup=256), dict(N=10, leaf=8, relax=16, maxsup=64, fem=3),
         dict(N=12, leaf=8, relax=37, maxsup=100, fem=3), dict(N=16, leaf=16, relax=64, maxsup=256, fem=3)]


@pytest.mark.parametrize("kw", CASES, ids=lambda kw: ("fem3" if kw.get("fem") else "poisson") + f"-{kw['N']}-ms{kw['maxsup']}")
def test_plan_matches_nesting_rule(kw, monkeypatch):
    monkeypatch.delenv("SLU_B200_SCHUR_DEPTH", raising=False)
    prob, _ = poisson_problem(**kw)
    ops = capi.plan(prob, schur_depth=1)
    seen = set()
    for depth in (1, 2, 3, 4):
        got = capi.schur_merge(prob, schur_depth=depth)
        assert got == _merge(prob, depth), (depth, got)
        st = capi.plan(prob, schur_depth=depth)
        assert (st.ops_fact, st.ops_schur, st.schur_bytes) == (ops.ops_fact, ops.ops_schur, ops.schur_bytes)
        assert st.lu_device_bytes == ops.lu_device_bytes and st.nlevels == ops.nlevels
        seen.add(got[0])
    assert capi.schur_merge(prob, schur_depth=1)[0] == 0
    assert max(seen) > 0, "no supernode chain on this problem"


def test_default_and_environment(monkeypatch):
    """options.reserved[6] = 0 takes the library default (4); SLU_B200_SCHUR_DEPTH overrides the option."""
    monkeypatch.delenv("SLU_B200_SCHUR_DEPTH", raising=False)
    prob, _ = poisson_problem(**CASES[0])
    assert capi.schur_merge(prob) == _merge(prob, 4)
    monkeypatch.setenv("SLU_B200_SCHUR_DEPTH", "1")
    assert capi.schur_merge(prob, schur_depth=3)[0] == 0
    monkeypatch.setenv("SLU_B200_SCHUR_DEPTH", "2")
    assert capi.schur_merge(prob, schur_depth=1) == _merge(prob, 2)


def test_off_where_unsupported(monkeypatch):
    """The int8 route and Pz > 1 plan without deferral."""
    monkeypatch.delenv("SLU_B200_SCHUR_DEPTH", raising=False)
    prob, _ = poisson_problem(**CASES[0])
    assert capi.schur_merge(prob, schur_depth=4, tc_slices=7)[0] == 0
    prob2, _ = poisson_problem(npdep=2, **CASES[0])
    assert capi.schur_merge(prob2, 0, schur_depth=4)[0] == 0
