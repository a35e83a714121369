"""Unsymmetric sparsity patterns stored as the reference stores them: every U block row cut to the exact skyline of
F = P A P^T (LUProblem.prune_u), so U columns start below their block's first row, columns and whole blocks of the
P (A + A^T) P^T structure are dropped, and panels carry no U index at all.

Two families, each with real and complex random-sign, row-diagonally dominant values (test_scaled_parity.mixed_values):
- band: a random unsymmetric band matrix in natural ordering, lower bandwidth larger than the upper one, sparse inside
  the band -- wide supernodes whose every U segment is short;
- upwind: 3D Poisson and FEM patterns with a random share of the one-sided couplings removed, nested-dissection
  ordered -- the tree and level structure.

Here, without a GPU: the skyline is exact against a dense unpivoted LU of F, filling a pruned problem puts F and
nothing else into the panels, the oracle on the pruned layout equals the oracle on the full layout, and the large
cases really have the shapes the GPU tests (test_gpu_unsym_skyline.py) claim to exercise."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle
from superlu_dist_b200 import LUProblem, hostlib
from superlu_dist_b200.problem import BC_HEADER, BR_HEADER, LB_DESCRIPTOR, UB_DESCRIPTOR
from test_scaled_parity import mixed_values, panel_coords
from util import rel_err, residual_probe

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
STAGE = 32 << 20            # elements per staging round of the skyline <-> dense-packed U conversion


# ----------------------------------------------------------------------------------------------------------- generators
def _csr(n, rows, cols, mag):
    a = sp.csr_matrix((mag, (rows, cols)), shape=(n, n))
    a.sum_duplicates()
    a.sort_indices()
    return a.indptr.astype(np.int32), a.indices.astype(np.int32), a.data.astype(np.float64)


def band_matrix(n, bl, bu, density, seed):
    """Pattern of a random band matrix: the diagonal, the first sub- and superdiagonal, and every other entry of the
    band -bl <= j - i <= bu with probability `density`.  -> (rowptr, colind, ones)"""
    rng = np.random.default_rng(seed)
    rows, cols = [np.arange(n)], [np.arange(n)]
    for d in range(-bl, bu + 1):
        if d == 0:
            continue
        i = np.arange(max(0, -d), min(n, n - d))
        keep = (rng.random(len(i)) < density) | (abs(d) == 1)
        rows.append(i[keep])
        cols.append(i[keep] + d)
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    return _csr(n, rows, cols, np.ones(len(rows)))


def upwind_matrix(N, frac, seed, fem=None):
    """Poisson 3D (fem=None) or FEM (dof = fem) pattern with a share `frac` of the couplings made one-sided: of each
    such pair (i, j), (j, i) one entry, picked at random, is removed.  -> (rowptr, colind, |values|), perm"""
    if fem:
        rp, ci, v = hostlib.fem3d(N, N, N, dof=fem)
        perm = hostlib.nd_order(N, dof=fem, leaf=8)
    else:
        rp, ci, v = hostlib.poisson3d(N)
        perm = hostlib.nd_order(N, leaf=8)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp)).astype(np.int64)
    ci = ci.astype(np.int64)
    pair = np.minimum(rows, ci) * n + np.maximum(rows, ci)
    _, inv = np.unique(pair, return_inverse=True)
    rng = np.random.default_rng(seed)
    cut, side = rng.random(inv.max() + 1) < frac, rng.random(inv.max() + 1) < 0.5
    drop = (rows != ci) & cut[inv] & ((rows < ci) == side[inv])
    return _csr(n, rows[~drop], ci[~drop], np.abs(v[~drop])), perm


# (family, matrix arguments, symbolic arguments); the small cases (n <= 1500) are dense-checkable
CASES = {
    "band_small": ("band", dict(n=1200, bl=60, bu=24, density=0.08, seed=1), dict(relax=16, maxsup=32, amalg=0.5)),
    "upwind_small": ("upwind", dict(N=10, frac=0.5, seed=2), dict(relax=8, maxsup=64, amalg=0.05)),
    "upwind_fem_small": ("upwind", dict(N=6, frac=0.8, seed=3, fem=3), dict(relax=8, maxsup=128, amalg=0.05)),
    "band": ("band", dict(n=40000, bl=300, bu=150, density=0.05, seed=4), dict(relax=64, maxsup=256, amalg=0.5)),
    "upwind": ("upwind", dict(N=24, frac=0.4, seed=5), dict(relax=32, maxsup=256, amalg=0.05)),
    "upwind_fem": ("upwind", dict(N=14, frac=0.8, seed=6, fem=2), dict(relax=32, maxsup=256, amalg=0.05)),
}
SMALL = ["band_small", "upwind_small", "upwind_fem_small"]
# the 27-point FEM couplings fill every U block that P (A + A^T) P^T has: those cases drop columns, not whole blocks
DROPS_BLOCKS = {"band_small", "upwind_small", "band", "upwind"}
LARGE = ["band", "upwind", "upwind_fem"]


@functools.lru_cache(maxsize=None)
def pattern(name):
    """-> (rowptr, colind, |values|, perm)"""
    family, mk, _ = CASES[name]
    if family == "band":
        rp, ci, v = band_matrix(**mk)
        return rp, ci, v, np.arange(len(rp) - 1, dtype=np.int32)
    (rp, ci, v), perm = upwind_matrix(**mk)
    return rp, ci, v, perm


def values(name, complex_=False, seed=0):
    rp, ci, v, _ = pattern(name)
    return mixed_values(rp, ci, v, seed, complex_)


def fill(prob, rp, ci, vals, z=0):
    """Layer z of prob holding vals (LUProblem.fill_layer takes float64 only: a complex matrix goes in part by part)."""
    lay = prob.add_layer(z) if z not in prob.layers else prob.layers[z]
    if np.iscomplexobj(lay.lval):       # a complex layer (refilled, or added after an earlier complex fill)
        lay.lval, lay.uval = np.zeros(len(lay.lval)), np.zeros(len(lay.uval))
    if not np.iscomplexobj(vals):
        prob.fill_layer(z, rp, ci, vals)
        return prob
    prob.fill_layer(z, rp, ci, np.ascontiguousarray(vals.real))
    lre, ure = lay.lval.copy(), lay.uval.copy()
    prob.fill_layer(z, rp, ci, np.ascontiguousarray(vals.imag))
    prob.dtype = np.dtype(np.complex128)
    lay.lval, lay.uval = lre + 1j * lay.lval, ure + 1j * lay.uval
    return prob


def make(name, vals=None, prune=True, npdep=1):
    """The problem of case `name`: the P (A + A^T) P^T structure, U cut to the exact skyline of F unless prune=False,
    every layer of the grid filled with vals (none when vals is None)."""
    rp, ci, v, perm = pattern(name)
    prob = LUProblem.from_matrix(rp, ci, v, perm, npdep=npdep, layers=(), **CASES[name][2])
    if prune:
        prob.prune_u(rp, ci)
    if vals is not None:
        for z in range(npdep):
            fill(prob, rp, ci, vals, z)
    return prob


def dense_f(name, vals):
    """F = P A P^T as a dense array."""
    rp, ci, _, perm = pattern(name)
    n = len(rp) - 1
    F = np.zeros((n, n), vals.dtype)
    rows = np.repeat(np.arange(n), np.diff(rp))
    F[perm[rows], perm[ci]] = vals
    return F


def dense_lu(F):
    """Unpivoted LU of F in place of a copy: strict lower part L (unit diagonal implied), upper part U."""
    a = F.copy()
    n = len(a)
    for k in range(n - 1):
        a[k + 1:, k] /= a[k, k]
        a[k + 1:, k + 1:] -= np.outer(a[k + 1:, k], a[k, k + 1:])
    return a


# ------------------------------------------------------------------------------------------------ host-side structure
def u_columns(prob):
    """Per U panel k: (columns, fstnz) of the stored columns (non-empty segments), in storage order."""
    xsup = np.asarray(prob.xsup)
    out = {}
    for k in range(prob.nsupers):
        if prob.uidx_off[k + 1] == prob.uidx_off[k]:
            continue
        idx = prob.uidx[prob.uidx_off[k]:prob.uidx_off[k + 1]]
        klst, u, cols, fst = int(xsup[k + 1]), BR_HEADER, [], []
        for _ in range(int(idx[0])):
            jb = int(idx[u])
            jf, jns = int(xsup[jb]), int(xsup[jb + 1] - xsup[jb])
            f = idx[u + UB_DESCRIPTOR:u + UB_DESCRIPTOR + jns]
            live = np.nonzero(f < klst)[0]
            cols.append(jf + live)
            fst.append(f[live])
            u += UB_DESCRIPTOR + jns
        out[k] = (np.concatenate(cols), np.concatenate(fst).astype(np.int64))
    return out


def l_rows(prob, s):
    """Rows of L panel s, diagonal block first."""
    idx, w, rows = prob.lidx[prob.lidx_off[s]:prob.lidx_off[s + 1]], BC_HEADER, []
    for _ in range(int(idx[0])):
        nb = int(idx[w + 1])
        rows.append(idx[w + LB_DESCRIPTOR:w + LB_DESCRIPTOR + nb])
        w += LB_DESCRIPTOR + nb
    return np.concatenate(rows)


def u_blocks(prob):
    """Number of U blocks with at least one stored column, over all panels."""
    xsup, nb = np.asarray(prob.xsup), 0
    for k, (cols, _) in u_columns(prob).items():
        nb += len(np.unique(np.searchsorted(xsup, cols, side="right") - 1))
    return nb


def skyline_counts(prob, full=None):
    """What a problem exercises, from its index arrays: U panels with short segments, those of them with m >= 96 and
    ncols >= 96 (updates on the schur_kernel_h tiles), U columns and blocks of the full structure `full` that pruning
    dropped, and the staging rounds of the skyline conversion (the greedy packing of slu_api.cu convert_u)."""
    xsup = np.asarray(prob.xsup, np.int64)
    ns = np.diff(xsup)
    m = np.asarray(prob.lidx)[np.asarray(prob.lidx_off)[:-1] + 1].astype(np.int64) - ns
    uc = u_columns(prob)
    short = [k for k, (cols, fst) in uc.items() if (fst > xsup[k]).any()]
    big = [k for k in short if m[k] >= 96 and len(uc[k][0]) >= 96]
    sky = [int(prob.uval_len[k]) for k in short]
    rounds = 0
    if sky:
        cap, i = max(max(sky), min(STAGE, 64 * max(sky))), 0
        while i < len(sky):
            used = 0
            while i < len(sky) and used + sky[i] <= cap:
                used += sky[i]
                i += 1
            rounds += 1
    out = dict(short_panels=len(short), big_tile_panels=len(big), nsupers=prob.nsupers,
               widest=int(ns.max()), staging_rounds=rounds, nnz_u=int(sum(ns[k] * len(c) for k, (c, _) in uc.items())))
    if full is not None:
        fc = u_columns(full)
        out["dropped_columns"] = sum(len(c) for c, _ in fc.values()) - sum(len(c) for c, _ in uc.values())
        out["dropped_blocks"] = u_blocks(full) - u_blocks(prob)
        out["dropped_panels"] = len(fc) - len(uc)
    return out


@functools.lru_cache(maxsize=None)
def counts(name):
    return skyline_counts(make(name), make(name, prune=False))


# ------------------------------------------------------------------------------------------------------------ the tests
@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_skyline_is_exact(name, complex_):
    """Against the dense unpivoted LU of F: U is exactly 0 above every stored column's fstnz and non-zero at it, and no
    non-zero of U (outside the diagonal blocks) lies in a column or block that pruning dropped."""
    prob = make(name)
    c = counts(name)
    assert c["short_panels"] > 0 and c["dropped_columns"] > 0, c
    assert c["dropped_blocks"] > 0 or name not in DROPS_BLOCKS, c
    LU = dense_lu(dense_f(name, values(name, complex_)))
    xsup = np.asarray(prob.xsup)
    stored = np.zeros(LU.shape, bool)
    for k in range(prob.nsupers):
        f, klst = int(xsup[k]), int(xsup[k + 1])
        stored[f:klst, f:klst] = True
    uc = u_columns(prob)
    lrows = [set(l_rows(prob, s).tolist()) for s in range(prob.nsupers)]
    ucols = [set(uc[s][0].tolist()) if s in uc else set() for s in range(prob.nsupers)]
    loose = 0
    for k, (cols, fst) in uc.items():
        f, klst = int(xsup[k]), int(xsup[k + 1])
        rows = np.arange(f, klst)[:, None]
        above = rows < fst[None, :]
        blk = LU[f:klst][:, cols]
        assert not blk[above].any(), f"panel {k}: a non-zero of U above a skyline start"
        # the start is tight: a non-zero of U, or a row an earlier update reaches through the stored structure (L keeps
        # P (A + A^T) P^T, so the L row of that update may hold explicit zeros)
        for q in np.nonzero(blk[fst - f, np.arange(len(cols))] == 0)[0]:
            r, j = int(fst[q]), int(cols[q])
            assert any(r in lrows[s] and j in ucols[s] for s in range(k)), f"panel {k}: column {j} starts too high"
            loose += 1
        stored[f:klst, cols] |= ~above
    upper = np.triu(np.ones(LU.shape, bool), 1)
    assert not (LU[upper & ~stored]).any(), "a non-zero of U outside the stored skyline"
    assert loose <= 0.2 * sum(len(c) for c, _ in uc.values()), loose


@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_fill_puts_f_and_nothing_else(name, complex_):
    """fill_layer on a pruned problem: the panels hold F exactly, and every stored value is an entry of F (nothing lands
    in another column's segment or outside the arena)."""
    vals = values(name, complex_)
    prob = make(name, vals)
    lay = prob.layers[0]
    F = dense_f(name, vals)
    assert np.array_equal(prob.dense(lay, False), F)
    assert len(lay.uval) == max(int(np.sum(prob.uval_len)), 1)
    assert np.count_nonzero(lay.lval) + np.count_nonzero(lay.uval) == np.count_nonzero(F)


_ABOVE = """
import sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
import numpy as np
from test_unsym_skyline_cpu import make, pattern, u_columns
name = {name!r}
rp, ci, v, perm = pattern(name)
prob = make(name)
k, (cols, fst) = next((k, c) for k, c in u_columns(prob).items() if (c[1] > prob.xsup[k]).any())
q = int(np.nonzero(fst > prob.xsup[k])[0][0])
iperm = np.argsort(perm)
i, j = int(iperm[prob.xsup[k]]), int(iperm[cols[q]])     # F(xsup[k], cols[q]) lies above the skyline start
rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
rows, cis = np.append(rows, i), np.append(ci, j)
o = np.lexsort((cis, rows))
rp2 = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=len(rp) - 1))]).astype(np.int32)
prob.add_layer(0)
print("filling", flush=True)
prob.fill_layer(0, rp2, cis[o].astype(np.int32), np.ones(len(o)))
print("filled", flush=True)
"""


def test_fill_refuses_entry_above_skyline():
    """An entry of A that falls above its U column's skyline start has no slot: sluh_fill_values stops with its "not in
    U structure" message instead of writing into another column's segment (run in a child process: it aborts)."""
    code = _ABOVE.format(tests=HERE, root=ROOT, name="band_small")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert "filling" in r.stdout and "filled" not in r.stdout, (r.stdout, r.stderr)
    assert r.returncode != 0 and "not in U structure" in r.stderr, r.stderr


def _u_map(pruned, full):
    """Positions in full's U arena of every value of pruned's U arena (same values layout on layer 0)."""
    _, _, pr, pc = panel_coords(pruned, pruned.layers[0])
    _, _, fr, fc = panel_coords(full, full.layers[0])
    n = pruned.n
    fk = fr * n + fc
    o = np.argsort(fk)
    q = o[np.searchsorted(fk[o], pr * n + pc)]
    assert np.array_equal(fk[q], pr * n + pc)
    return q


@pytest.mark.parametrize("name", SMALL + ["upwind"])
@pytest.mark.parametrize("complex_", [False, True], ids=["double", "complex"])
def test_oracle_pruned_equals_full(name, complex_):
    """The oracle on the pruned layout against the oracle on the full P (A + A^T) P^T layout of the same matrix: equal
    on the shared slots, the full layout's extra U slots exactly 0, and ||LU - F|| / ||F|| < 1e-13."""
    vals = values(name, complex_)
    pruned, full = make(name, vals), make(name, vals, prune=False)
    pre = pruned.layers[0].copy()
    info, ops, _ = oracle.factor(pruned)
    finfo, fops, _ = oracle.factor(full)
    assert info == finfo == 0
    assert ops < fops                       # the pruned layout skips the updates of the dropped columns
    lp, lf = pruned.layers[0], full.layers[0]
    assert rel_err(lp.lval, lf.lval) < 1e-13
    q = _u_map(pruned, full)
    assert rel_err(lp.uval, lf.uval[q]) < 1e-13
    extra = np.ones(len(lf.uval), bool)
    extra[q] = False
    assert not lf.uval[extra].any()
    if not complex_:
        every = np.ones(pruned.nsupers, bool)
        assert residual_probe(pruned, [(pre, every)], [(lp, every)]) < 1e-13


@pytest.mark.parametrize("name", LARGE)
def test_large_cases_have_the_claimed_shape(name):
    """The GPU cases exercise what they claim: short-skyline panels, short-skyline panels on the big Schur tiles,
    dropped columns and blocks, and (the band) more than one staging round of the skyline conversion."""
    c = counts(name)
    assert c["short_panels"] > 0 and c["big_tile_panels"] > 0, c
    assert c["dropped_columns"] > 0, c
    assert c["dropped_blocks"] > 0 or name not in DROPS_BLOCKS, c
    if name == "band":
        assert c["staging_rounds"] >= 2 and c["widest"] == 256, c
