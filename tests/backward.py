"""Componentwise backward error of the kernels, factorizations and solves (test infrastructure, imported like util).

A correctly rounded algorithm of the same shape as the reference's meets each bound here whatever the condition number
of its input, so these checks need no oracle and stay sharp on graded, indefinite and tiny-pivot inputs, where the
normwise checks (rel_err against the oracle) are either blind to small entries or too loose to mean anything.

Every ratio is |R| / D elementwise.  R is computed in extended precision (np.longdouble: 64-bit significand on x86), so
that the residual of a double-precision result is exact to far below the bounds; D, a sum of non-negative terms, is
accurate to a few ulps in double.  R != 0 where D == 0 counts as infinity: a
write to a position that no product touches fails.  In doublecomplex |.| is the modulus and every bound doubles.

    operation                  residual R                     scale D                 bound
    diag LU (k_diag_lu)        A - L U                        |L| |U|                 4 ns u
    trsm L case (X U = B)      X U - B                        |X| |U|                 4 ns u
    trsm U case (L X = B)      L X - B                        |L| |X|                 4 ns u
    gemm_sub (C - A B)         C_out - (C - A B)              |C| + |A| |B|           2 (k + 1) u
    factorization              F - L U on pattern(F, L U)     |L| |U|                 4 k_max u
    solve, op = N / T / H      b - op(L U) x, per row         op(|L| |U|) |x|         4 k_max u
    selected inversion         per step of each supernode: the table of the last section

u = 2^-53.  k_max is the largest panel height (nsupr) of the problem.  The bounds are fixed formulas in u: none is
tuned to what a GPU returns.  Pivots replaced by +-thresh (static pivoting) are excluded from the factorization ratio
at their own diagonal position; the callers check that their count is the kernel's tiny-pivot count."""
import numpy as np
import scipy.sparse as sp

from test_scaled_parity import panel_coords

U = 2.0 ** -53
LD, CLD = np.longdouble, np.clongdouble


def ext(a):
    """a in extended precision (long double, complex long double for complex a)"""
    return a.astype(CLD if np.iscomplexobj(a) else LD)


def cfactor(dtype):
    """2 for doublecomplex, 1 for double: every bound doubles in complex"""
    return 2 if np.dtype(dtype).kind == "c" else 1


def ratio(r, d):
    """max |r| / d elementwise (arrays of the same shape, d >= 0); r != 0 with d == 0 is infinity, 0 / 0 is 0"""
    r = np.abs(np.asarray(r))
    d = np.asarray(d)
    if r.size == 0:
        return 0.0
    bad = (d == 0) & (r != 0)
    q = np.where(d > 0, r / np.where(d > 0, d, 1), 0)
    return float(np.inf) if bad.any() else float(q.max())


# ------------------------------------------------------------------------------------------------- kernel inputs
# The widths cross the 16-column blocks of the TRSM and its inverses, the 32-column slabs and the 65..256 range of the
# cluster diagonal LU, and the 64-row T chunks; the vector counts cross the 32-vector TRSM strip.
WIDTHS = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 96, 97, 255, 256, 257, 416, 417, 512]
ZWIDTHS = [w for w in WIDTHS if w <= 256]
VECS = [1, 31, 32, 33, 95, 1000]
# dominant: the inputs of test_gpu_kernels.py.  nondom: |u_ii| in [0.5, 2], off-diagonal entries that outweigh it
# (|l| <= 1 in the unit lower factor).  graded: rows scaled log-uniformly over [1e-6, 1], the first 16 columns swept over
# the whole range.  tiny: exact tiny pivots at block and slab boundaries.  scaled: rows and columns scaled by powers of
# two up to 2^+-300.  zpivots (complex): pivots with |Im| / |Re| = 1e+-12, purely imaginary ones and |pivot| = 2^+-600,
# where a naive |a|^2 overflows.
FAMILIES = ["dominant", "nondom", "graded", "tiny", "scaled"]
ZFAMILIES = FAMILIES + ["zpivots"]
TINY_COLS = (0, 15, 16, 31, 32, 63, 64, 255, 256)
TINY_PIVOT = 1e-30      # planted in the diagonal LU's input, below THRESH: replaced
THRESH = 2.0 ** -26     # the replacement value; the triangles of the TRSM take it as their tiny pivots


def vecs_for(ns, family):
    """One vector count per (width, family), rotating through VECS; 1000 vectors only up to 128 columns (95 past it),
    which keeps every extended-precision residual under a second"""
    m = VECS[(WIDTHS.index(ns) + ZFAMILIES.index(family)) % len(VECS)]
    return 95 if m == 1000 and ns > 128 else m


def _rand(rng, shape, z, kind="normal"):
    draw = (lambda: rng.standard_normal(shape)) if kind == "normal" else (lambda: rng.uniform(-1.0, 1.0, shape))
    return draw() + 1j * draw() if z else draw()


def _pivots(rng, ns, z):
    mag = rng.uniform(0.5, 2.0, ns)
    return mag * (np.exp(2j * np.pi * rng.uniform(size=ns)) if z else rng.choice([-1.0, 1.0], ns))


def _special(ns, family):
    """columns whose pivot is planted (their row of the unit lower factor is zero left of the diagonal)"""
    if family == "tiny":
        return [c for c in TINY_COLS if c < ns]
    if family == "zpivots":
        return list(range(0, ns, 3))
    return []


def _graded(rng, ns):
    d = 10.0 ** rng.uniform(-6.0, 0.0, ns)
    w = min(16, ns)
    d[:w] = 10.0 ** (-6.0 * np.arange(w) / 15)
    return d


def upper(family, ns, rng, z, pivot_tiny=THRESH, scale_rows=True):
    """An upper triangle of `family` (the U of X U = B, or U0 of a diagonal LU input).  zpivots: scale_rows puts the
    2^+-600 moduli on the whole row (a TRSM stays in range: one column of X scales), else on the pivot alone (the
    diagonal LU's multipliers below it stay O(1), and the reciprocal of the pivot must not overflow)."""
    if family == "dominant":
        return np.triu(_rand(rng, (ns, ns), z)) + ns * np.eye(ns)
    u = np.triu(_rand(rng, (ns, ns), z, "uniform"), 1) / np.sqrt(ns)
    p = _pivots(rng, ns, z)
    rs = np.ones(ns)
    if family == "graded":
        rs = _graded(rng, ns)
    elif family == "scaled":
        rs = 2.0 ** rng.integers(-300, 301, ns)
    elif family == "tiny":
        for c in _special(ns, family):
            p[c] = pivot_tiny * (-1.0 if c % 2 else 1.0) * (np.exp(0.25j * np.pi) if z else 1.0)
    elif family == "zpivots":
        kinds = [np.exp(1j * np.arctan(1e-12)), np.exp(1j * np.arctan(1e12)), 1j, -1j, 1.0, 1.0]
        scale = [1.0, 1.0, 1.0, 1.0, 2.0 ** 600, 2.0 ** -600]
        for t, c in enumerate(_special(ns, family)):
            p[c] = abs(p[c]) * kinds[t % 6] * (1.0 if scale_rows else scale[t % 6])
            rs[c] = scale[t % 6] if scale_rows else 1.0
            u[:c, c] = 0.0   # with row c of L0 zero, the pivot of A = L0 U0 is exactly p[c] and nothing cancels
    u = u + np.diag(p)
    if family == "scaled":
        u = u * 2.0 ** rng.integers(-300, 301, ns)[None, :]
    return rs[:, None] * u


def unit_lower(family, ns, rng, z, special=()):
    """A unit lower triangle of `family` (the L of L X = B, or L0 of a diagonal LU input); rows in `special` are zero
    left of the diagonal"""
    if family == "dominant":
        return np.tril(_rand(rng, (ns, ns), z), -1) / ns + np.eye(ns)
    lo = np.tril(_rand(rng, (ns, ns), z, "uniform"), -1) / np.sqrt(ns)
    lo[list(special)] = 0.0
    if family == "graded":
        d = _graded(rng, ns)
        lo = d[:, None] * lo / d[None, :]
    elif family == "scaled":
        d = 2.0 ** rng.integers(-150, 151, ns)
        lo = d[:, None] * lo / d[None, :]
    return lo + np.eye(ns)


def diag_lu_input(family, ns, extra, seed, z=False):
    """(ns + extra) x ns: A = L0 U0 on top (randn + ns I for dominant), random rows below.  scaled: Dr (L0 U0) Dc with
    the non-dominant L0 and U0, whose LU is Dr L0 Dr^-1 and Dr U0 Dc exactly in binary floating point."""
    rng = np.random.default_rng(seed)
    if family == "dominant":
        top = _rand(rng, (ns, ns), z) + ns * np.eye(ns)
    elif family == "scaled":
        top = unit_lower("nondom", ns, rng, z) @ upper("nondom", ns, rng, z)
        top = 2.0 ** rng.integers(-300, 301, ns)[:, None] * top * 2.0 ** rng.integers(-300, 301, ns)[None, :]
    else:
        top = unit_lower(family, ns, rng, z, _special(ns, family)) @ upper(family, ns, rng, z, TINY_PIVOT, False)
    return np.vstack([top, _rand(rng, (extra, ns), z)])


def trsm_l_input(family, ns, m, seed, z=False):
    """(U, B) of X U = B; B's rows scaled by powers of two up to 2^+-300 in the scaled family"""
    rng = np.random.default_rng(seed)
    u = upper(family, ns, rng, z)
    b = _rand(rng, (m, ns), z)
    if family == "scaled":
        b = b * 2.0 ** rng.integers(-300, 301, m)[:, None]
    return u, b


def trsm_u_input(family, ns, nc, seed, z=False):
    """(L, B) of L X = B (the unit lower triangle of the first; its diagonal is not read)"""
    rng = np.random.default_rng(seed)
    lo = unit_lower(family, ns, rng, z)
    b = _rand(rng, (ns, nc), z)
    if family == "scaled":
        b = b * 2.0 ** rng.integers(-300, 301, nc)[None, :]
    return lo, b


# Consistent right-hand sides: B = X T formed in extended precision and rounded, X uniform in [-1, 1], the kind of B a
# factorization hands the panel TRSM (B = L U_kk with moderate L).  A random B makes X as large as the conditioning of T
# allows, and then even a product with an explicit inverse of T_jj passes; with a consistent B that product has a
# backward error that grows with cond(T_jj), while substitution's does not.  One column is planted per chosen 16-column
# block (the first, a middle and the last, possibly partial, one) at in-block offsets 1, 7 and 14, rotated by ns mod 3.
DELTAS = [1e-4, 1e-8, 1e-12]
CWIDTHS = [w for w in WIDTHS if w >= 16]
ZCWIDTHS = [w for w in ZWIDTHS if w >= 16]
CVECS = 33   # crosses the 32-vector TRSM strip


def consistent_positions(ns):
    nb = (ns + 15) // 16
    offs = np.roll((1, 7, 14), ns % 3)
    return sorted({min(16 * blk + int(o), ns - 1) for blk, o in zip(sorted({0, nb // 2, nb - 1}), offs)})


def trsm_l_consistent(ns, m, delta, positions, seed, z=False):
    """(U, B) of X U = B: U upper, off-diagonal uniform in [-1, 1], pivots of modulus in [1, 2] (random phase in complex)
    but delta (times the phase) at `positions`"""
    rng = np.random.default_rng(seed)
    u = np.triu(_rand(rng, (ns, ns), z, "uniform"), 1)
    d = rng.uniform(1.0, 2.0, ns)
    d[list(positions)] = delta
    u = u + np.diag(d * np.exp(2j * np.pi * rng.uniform(size=ns)) if z else d * rng.choice([-1.0, 1.0], ns))
    x = _rand(rng, (m, ns), z, "uniform")
    return u, (ext(x) @ ext(u)).astype(u.dtype)


def trsm_u_consistent(ns, nc, delta, positions, seed, z=False):
    """(L, B) of L X = B: L unit lower, multipliers uniform in [-1, 1], those of the columns at `positions` times
    delta^-1/2 (the multipliers below a pivot of delta in a factor whose |L| |U| stays moderate)"""
    rng = np.random.default_rng(seed)
    lo = np.tril(_rand(rng, (ns, ns), z, "uniform"), -1)
    lo[:, list(positions)] *= delta ** -0.5
    lo = lo + np.eye(ns)
    x = _rand(rng, (ns, nc), z, "uniform")
    return lo, (ext(lo) @ ext(x)).astype(lo.dtype)


GEMM_SHAPES = [(1, 1, 1), (33, 31, 7), (96, 97, 17), (128, 130, 100), (257, 131, 137), (200, 97, 256), (129, 300, 513)]
GEMM_FAMILIES = ["random", "cancel", "scaled"]


def gemm_input(family, m, n, k, seed, z=False):
    """(A, B, C) of C - A B.  cancel: C = fl(A B) plus a perturbation of 2^-40 of it; scaled: rows of A and C by 2^+-200"""
    rng = np.random.default_rng(seed)
    a, b, c = _rand(rng, (m, k), z), _rand(rng, (k, n), z), _rand(rng, (m, n), z)
    if family == "cancel":
        c = a @ b
        c = c + 2.0 ** -40 * c * rng.uniform(-1.0, 1.0, c.shape)
    elif family == "scaled":
        r = 2.0 ** rng.integers(-200, 201, m)[:, None]
        a, c = a * r, c * r
    return a, b, c


# ---------------------------------------------------------------------------------------------------- restatements
def lu_nopivot_ld(a, thresh=None):
    """Right-looking LU without pivoting in extended precision, rounded to the input's dtype; tiny pivots replaced by
    +-thresh as the kernels do (pdgstrf2.c: |p| < thresh; pzgstrf2.c: |re| + |im| < thresh with both parts non-zero)
    -> (factored block, replaced count)"""
    w = ext(np.array(a))
    ns, tiny, z = w.shape[1], 0, np.iscomplexobj(a)
    for j in range(ns):
        p = w[j, j]
        small = (abs(p.real) + abs(p.imag) < thresh and p.real != 0 and p.imag != 0) if z else abs(p) < thresh
        if thresh is not None and small:
            w[j, j] = -thresh if p.real < 0 else thresh
            tiny += 1
        if w[j, j] != 0:
            w[j + 1:ns, j] /= w[j, j]
        w[j + 1:ns, j + 1:] -= np.outer(w[j + 1:ns, j], w[j, j + 1:])
    return w.astype(a.dtype), tiny


def _inv_upper16(t):
    """Inverse of an upper triangle, column by column from the diagonal up, dividing by the pivot (diag_inv_kernel)"""
    m = t.shape[0]
    x = np.zeros_like(t)
    for r in range(m - 1, -1, -1):
        s = (np.arange(m) == r).astype(t.dtype)
        for q in range(r + 1, m):
            s = s - t[r, q] * x[q]
        x[r] = np.where(np.arange(m) >= r, s / t[r, r], 0)
    return x


def _inv_unit_lower16(lo):
    """Inverse of a unit lower triangle, column by column downwards (diag_inv_kernel)"""
    m = lo.shape[0]
    x = np.eye(m, dtype=lo.dtype)
    for r in range(1, m):
        s = np.zeros(m, lo.dtype)
        for q in range(r):
            s = s - lo[r, q] * x[q]
        x[r] = np.where(np.arange(m) < r, s, x[r])
    return x


def trsm_blocked(t, b, unit, refine=1):
    """trsm_kernel's algorithm in NumPy: Y <- Y T^-1 blocked by 16 columns; with R = Y_j - sum_{p<j} Y_p T_pj and the
    explicit 16 x 16 inverse of diag_inv_kernel, X = R inv(T_jj), then `refine` correction steps X += (R - X T_jj) inv.
    unit: T = L^T of a unit lower L (the U case; the diagonal of T is taken as 1).  refine=0 is the plain product with
    the inverse, which is not backward stable on consistent right-hand sides: kept to show that the tests see it."""
    ns = t.shape[0]
    y = b.copy()
    for j0 in range(0, ns, 16):
        j1 = min(ns, j0 + 16)
        tjj = np.triu(t[j0:j1, j0:j1], 1) + np.eye(j1 - j0) if unit else np.triu(t[j0:j1, j0:j1])
        inv = _inv_unit_lower16(tjj.T).T if unit else _inv_upper16(tjj)
        r = y[:, j0:j1] - y[:, :j0] @ t[:j0, j0:j1]
        x = r @ inv
        for _ in range(refine):
            x = x + (r - x @ tjj) @ inv
        y[:, j0:j1] = x
    return y


# --------------------------------------------------------------------------------------------------- dense (kernels)
def diag_lu_ratio(a, out, thresh=None):
    """k_diag_lu: A (ns + extra) x ns in, the factored block out -> (ratio on the ns x ns block, replaced pivots).
    Diagonal positions where |u_kk| == thresh (pivots replaced by +-thresh) are excluded."""
    ns = a.shape[1]
    L = np.tril(out[:ns], -1) + np.eye(ns)
    Uf = np.triu(out[:ns])
    R = ext(a[:ns]) - ext(L) @ ext(Uf)
    D = np.abs(L) @ np.abs(Uf)
    rep = np.zeros(ns, bool) if thresh is None else np.abs(np.diag(out[:ns])) == thresh
    R[np.diag_indices(ns)] = np.where(rep, 0, np.diag(R))
    return ratio(R, D), int(rep.sum())


def trsm_l_ratio(u, b, x):
    """X U = B, U the upper triangle of u (non-unit)"""
    Ut = np.triu(u)
    return ratio(ext(x) @ ext(Ut) - ext(b), np.abs(x) @ np.abs(Ut))


def trsm_u_ratio(lo, b, x):
    """L X = B, L the strict lower triangle of lo plus the unit diagonal"""
    Lt = np.tril(lo, -1) + np.eye(lo.shape[0])
    return ratio(ext(Lt) @ ext(x) - ext(b), np.abs(Lt) @ np.abs(x))


def gemm_sub_ratio(a, b, c, out):
    return ratio(ext(out) - (ext(c) - ext(a) @ ext(b)), np.abs(c) + np.abs(a) @ np.abs(b))


def kernel_bound(ns, dtype):
    return 4 * ns * U * cfactor(dtype)


def gemm_bound(k, dtype):
    return 2 * (k + 1) * U * cfactor(dtype)


# ---------------------------------------------------------------------------------------------- sparse (factorizations)
def _csr(rows, cols, vals, n):
    m = sp.csr_matrix((vals, (rows, cols)), shape=(n, n))
    m.sum_duplicates()
    return m


def panel_matrix(prob, layer):
    """The unfactored layer (F = P A P^T as the panels hold it) as CSR"""
    lrow, lcol, urow, ucol = panel_coords(prob, layer)
    lk, uk = lrow >= 0, urow >= 0
    return _csr(np.concatenate([lrow[lk], urow[uk]]), np.concatenate([lcol[lk], ucol[uk]]),
                np.concatenate([layer.lval[lk], layer.uval[uk]]), prob.n)


def factors(prob, layer, n_elim=None):
    """(L, U) of one factored layer as CSR: L unit lower (the identity added), U upper, the walk of LUProblem.dense.
    n_elim: only the first n_elim columns were eliminated (a partial factorization); the panels of the later columns
    are left out, and L gets the identity there."""
    n = prob.n
    n_elim = n if n_elim is None else n_elim
    lrow, lcol, urow, ucol = panel_coords(prob, layer)
    lk = (lrow >= 0) & (lcol < n_elim)
    uk = (urow >= 0) & (urow < n_elim)
    lr, lc, lv = lrow[lk], lcol[lk], layer.lval[lk]
    low = lr > lc
    eye = np.arange(n)
    L = _csr(np.concatenate([lr[low], eye]), np.concatenate([lc[low], eye]),
             np.concatenate([lv[low], np.ones(n, lv.dtype)]), n)
    Uf = _csr(np.concatenate([lr[~low], urow[uk]]), np.concatenate([lc[~low], ucol[uk]]),
              np.concatenate([lv[~low], layer.uval[uk]]), n)
    return L, Uf


def csr_values(rp, ci, vals, perm, n, rperm=None):
    """F(perm[rperm[i]], perm[j]) = a_ij of the CSR matrix (rperm: row permutation applied first, None the identity)"""
    rows = np.repeat(np.arange(n), np.diff(rp))
    perm = np.asarray(perm)
    ri = rows if rperm is None else np.asarray(rperm)[rows]
    return _csr(perm[ri], perm[np.asarray(ci)], np.asarray(vals), n)


def k_max(prob):
    """The largest panel height nsupr: every dot product of the factorization and the solves is at most this long"""
    return int(np.asarray(prob.lidx)[np.asarray(prob.lidx_off)[:-1] + 1].max())


def factor_bound(prob):
    return 4 * k_max(prob) * U * cfactor(prob.dtype)


def _keys(m):
    m = m.tocoo()
    return m.row.astype(np.int64) * m.shape[1] + m.col, m.data


def factor_ratio(F, L, Uf, thresh=None):
    """max |F - L U| / (|L| |U|) over pattern(F) and pattern(L U), in extended precision -> (ratio, replaced pivots).
    thresh: exclude the diagonal positions where |u_kk| == thresh (pivots replaced by +-thresh)."""
    R = (ext(F).tocsr() - ext(L).tocsr() @ ext(Uf).tocsr()).tocsr()
    D = (abs(L) @ abs(Uf)).tocsr()
    d = Uf.diagonal()
    rep = np.zeros(F.shape[0], bool) if thresh is None else np.abs(d) == thresh
    rk, rv = _keys(R)
    n = F.shape[0]
    drop = np.isin(rk, np.nonzero(rep)[0] * (n + 1))
    rk, rv = rk[~drop], rv[~drop]
    dk, dv = _keys(D)
    o = np.argsort(dk)
    dk, dv = dk[o], dv[o]
    q = np.minimum(np.searchsorted(dk, rk), max(len(dk) - 1, 0))
    hit = (dk[q] == rk) if len(dk) else np.zeros(len(rk), bool)
    den = np.where(hit, dv[q] if len(dv) else 0, 0)
    return ratio(rv, den), int(rep.sum())


def _op(M, trans):
    return {"N": M, "T": M.T, "H": M.conj().T}[trans]


def solve_ratio(L, Uf, x, b, trans="N"):
    """max over right-hand sides and rows of |b - op(L U) x| / (op(|L| |U|) |x|); x, b: (n,) or (nrhs, n)"""
    Le, Ue = ext(L).tocsr(), ext(Uf).tocsr()
    x, b = np.atleast_2d(x).T, np.atleast_2d(b).T
    X, B = ext(x), ext(b)
    if trans == "N":
        R = B - Le @ (Ue @ X)
        D = abs(L) @ (abs(Uf) @ np.abs(x))
    else:
        R = B - _op(Ue, trans) @ (_op(Le, trans) @ X)
        D = abs(Uf).T @ (abs(L).T @ np.abs(x))
    return ratio(R, D)


# ------------------------------------------------------------------------------------------ factorization problems
# Poisson 12^3 (maxsup 128); the 256-column top separator of Poisson 16^3; fem 6^3 x 3 (supernodes up to 200 columns);
# supernodes of at most 8 columns, so that the 64-column Schur tiles span eight or more destination panels (Poisson
# 16^3: 1524 such tiles, the layout of test_gpu_schur_destinations.py at a size whose residual takes seconds).
PROBLEMS = {"poisson12": dict(N=12, leaf=8, relax=16, maxsup=128),
            "top256": dict(N=16, leaf=16, relax=32, maxsup=256),
            "fem6": dict(N=6, leaf=4, relax=8, maxsup=200, fem=3),
            "narrow": dict(N=16, leaf=8, relax=8, maxsup=8)}
ZPROBLEMS = {"z32": dict(N=8, leaf=4, relax=8, maxsup=32),
             "z200": dict(N=6, leaf=4, relax=8, maxsup=200, fem=3)}
# a dyadic shift of Poisson 12^3 between two eigenvalues (test_inertia_cpu.gap_shifts): mixed-sign, small pivots
SHIFT_N, SHIFT_KW = 12, dict(N=12, leaf=8, relax=16, maxsup=128)


def shift_sigma():
    from test_inertia_cpu import gap_shifts, spectrum
    return gap_shifts(spectrum(SHIFT_N), 7)[3]


# Planted factors: F = fl(L0 U0) with moderate L0 and U0 on the panel pattern, so that every panel TRSM of the
# factorization of F gets a consistent right-hand side; small pivots are planted in the widest supernodes (PLANTED_DELTA).
# "w512": fem 8^3 x 3 relaxed into supernodes of 512, 384, 288 and 256 columns (panels up to 768 rows).
PLANTED = {"top256": PROBLEMS["top256"], "fem6": PROBLEMS["fem6"],
           "w512": dict(N=8, leaf=8, relax=512, maxsup=512, fem=3)}
ZPLANTED = {"z200": ZPROBLEMS["z200"]}
PLANTED_DELTA = 1e-6     # a computed pivot of delta perturbs what follows by ~ u / delta: keep the others planted
PLANTED_MULT = 1e4       # the multipliers of the scaled columns (their U rows scaled by its inverse)
PLANTED_NODES = 3        # the widest supernodes get the planted pivots


def planted_nodes(prob, count=PLANTED_NODES):
    ns = np.diff(np.asarray(prob.xsup))
    return sorted(np.argsort(-ns, kind="stable")[:count].tolist())


def plant_factors(prob, delta=PLANTED_DELTA, mult=PLANTED_MULT, seed=0, nodes=None):
    """L0 (unit lower) and U0 (upper) on the panel pattern of layer 0: entries uniform in [-1, 1] scaled by 1 / sqrt of
    the supernode's width, pivots of modulus in [1, 2] with random signs (phases in complex).  In each supernode of
    `nodes` (default: the widest), at the positions consistent_positions(ns) picks: a pivot of delta (an ill-conditioned
    U_kk for the L-panel TRSM); and two columns on, multipliers scaled by mult and the U row beside the pivot by 1 / mult
    (an ill-conditioned L_kk for the U-panel TRSM; that column of L0 times that row of U0 stays O(1)).  Writes
    F = fl(L0 U0) into layer 0 and checks that no entry of F falls outside the panels.  -> F as CSR."""
    lay = prob.layers[0]
    z = np.iscomplexobj(lay.lval)
    rng = np.random.default_rng(seed)
    lrow, lcol, urow, ucol = panel_coords(prob, lay)
    xsup = np.asarray(prob.xsup)
    n = prob.n
    width = np.diff(xsup)[np.searchsorted(xsup, np.arange(n), side="right") - 1]
    lk, uk = lrow >= 0, urow >= 0
    rows = np.concatenate([lrow[lk], urow[uk]])
    cols = np.concatenate([lcol[lk], ucol[uk]])
    vals = _rand(rng, len(rows), z, "uniform") / np.sqrt(width[np.minimum(rows, cols)])
    piv = rng.uniform(1.0, 2.0, n) * (np.exp(2j * np.pi * rng.uniform(size=n)) if z else rng.choice([-1.0, 1.0], n))
    lscale, uscale = np.ones(n), np.ones(n)
    for k in (planted_nodes(prob) if nodes is None else nodes):
        f, ns = int(xsup[k]), int(xsup[k + 1] - xsup[k])
        for p in consistent_positions(ns):
            piv[f + p] *= delta
            q = f + (p + 2) % ns
            lscale[q], uscale[q] = mult, 1.0 / mult
    low, dia = rows > cols, rows == cols
    vals = np.where(low, vals * lscale[cols], vals * uscale[rows])
    vals[dia] = piv[rows[dia]]
    L0 = _csr(np.concatenate([rows[low], np.arange(n)]), np.concatenate([cols[low], np.arange(n)]),
              np.concatenate([vals[low], np.ones(n, vals.dtype)]), n)
    U0 = _csr(rows[~low], cols[~low], vals[~low], n)
    F = (ext(L0) @ ext(U0)).astype(vals.dtype).tocsr()
    assert np.isin(_keys(F)[0], rows.astype(np.int64) * n + cols).all(), "an entry of L0 U0 falls outside the panels"
    lay.lval[lk] = np.asarray(F[lrow[lk], lcol[lk]]).ravel()
    lay.uval[uk] = np.asarray(F[urow[uk], ucol[uk]]).ravel()
    return F


def to_csr(F, perm):
    """The CSR (rowptr, colind, values) of A = P^T F P, perm[old] = new: what fill_csr takes to put F into the panels"""
    perm = np.asarray(perm)
    A = F.tocsr()[perm][:, perm].tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data


def panel_trsm_ratios(prob, L, Uf, refine, nodes=None):
    """The panel TRSMs of a factorization restated on its factors: for supernode k with columns f..l, X_L U_kk = B_L and
    L_kk X_U = B_U with X_L, X_U the L rows below and the U columns right of the diagonal block, and B formed from them
    in extended precision; trsm_blocked(refine) solves.  -> the largest ratio / kernel_bound(ns) of each case"""
    xsup = np.asarray(prob.xsup)
    L, Uf = L.tocsc(), Uf.tocsr()
    worst = [0.0, 0.0]
    for k in (range(prob.nsupers) if nodes is None else nodes):
        f, l = int(xsup[k]), int(xsup[k + 1])
        ukk = Uf[f:l, f:l].toarray()
        lkk = L[f:l, f:l].toarray()
        xl = L[l:, f:l].tocsr()
        xl = xl[np.diff(xl.indptr) > 0].toarray()
        xu = Uf[f:l, l:].tocsc()
        xu = xu[:, np.diff(xu.indptr) > 0].toarray()
        bound = kernel_bound(l - f, prob.dtype)
        if len(xl):
            b = (ext(xl) @ ext(ukk)).astype(xl.dtype)
            worst[0] = max(worst[0], trsm_l_ratio(ukk, b, trsm_blocked(ukk, b, False, refine)) / bound)
        if xu.shape[1]:
            b = (ext(lkk) @ ext(xu)).astype(xu.dtype)
            worst[1] = max(worst[1], trsm_u_ratio(lkk, b, trsm_blocked(lkk.T, b.T, True, refine).T) / bound)
    return tuple(worst)


def kkt_matrix():
    """The KKT matrix of test_gpu_static_pivot.py: zero (2, 2) block, no unpivoted LU in the natural order"""
    from test_static_pivot_cpu import kkt
    return kkt(16, 40, 3)


KKT_THRESH = 0.625   # above the smallest pivots of the matched, scaled KKT matrix (0.57..): some are replaced


# ------------------------------------------------------------------------------------------------ selected inversion
# H = F^-T supernode by supernode (oracle/selinv.py, slu_selinv.cu).  For supernode K with sub-diagonal rows R (m of them),
# packed U columns C (ncols) and M = H(R, C) gathered from the returned H, each step solves its own equations:
#
#    step     residual R                                           scale D                                          bound
#    H(R,K)   H(R,K) U_KK^T + M U_KC^T                             |H(R,K)| |U_KK|^T + |M| |U_KC|^T                  4 (ns + ncols) u
#    H(K,C)   L_KK^T H(K,C) + L_RK^T M                             |L_KK|^T |H(K,C)| + |L_RK|^T |M|                  4 (ns + m) u
#    H(K,K)   L_KK^T H(K,K) U_KK^T - I + L_RK^T H(R,K) U_KK^T      |L_KK|^T |H(K,K)| |U_KK|^T + I                    8 (ns + m) u
#                                                                  + |L_RK|^T (|H(R,K)| |U_KK|^T + |M| |U_KC|^T)
#
# Each is a product of length ncols or m (its rounding is covered by the terms with M or L_RK) and one triangular solve of
# length ns (a substitution's backward error is within the terms with the solved block); H(K,K) takes two solves and the
# product that forms its right-hand side, hence twice the constant.  Doubled in complex, as every bound here.  H(K,C) is
# checked where it is stored: row i of column j from the column's skyline start on (rows above it are not kept, and
# L_KK^T, upper triangular, takes the stored rows from the stored rows only).
SELINV_STEPS = ("H(R,K)", "H(K,C)", "H(K,K)")


def _selinv_node(P, lval, uval, k):
    """(ns, Lkk unit lower, Ukk upper, Lrk, Ukc dense-packed, R, C) of supernode k of the factors lval / uval"""
    f, ns = int(P.xsup[k]), int(P.xsup[k + 1] - P.xsup[k])
    Lp = P.lpanel(lval, k)
    return (ns, np.tril(Lp[:ns], -1) + np.eye(ns), np.triu(Lp[:ns]), Lp[ns:], P.upanel(uval, k),
            P.lrows[k][ns:], P.ucols[k])


def _gather_m(P, hl, hu, R, C):
    return P.gather(hl, hu, R, C) if len(R) and len(C) else np.zeros((len(R), len(C)), hl.dtype)


def selinv_ratios(prob, layer, hl, hu):
    """The three steps of every supernode of the factors in `layer`, on H as returned (hl, hu shaped like layer.lval /
    layer.uval) -> (the largest ratio / bound of each step, the largest ratio of each step)"""
    from oracle.selinv import _Panels
    P = _Panels(prob, layer)
    cf = cfactor(layer.lval.dtype)
    scaled, raw = np.zeros(3), np.zeros(3)
    for k in np.nonzero(layer.held)[0]:
        ns, Lkk, Ukk, Lrk, Ukc, R, C = _selinv_node(P, layer.lval, layer.uval, k)
        f, m, nc = int(P.xsup[k]), len(R), len(C)
        Hp = P.lpanel(hl, k)
        Hkk, Hrk = Hp[:ns], Hp[ns:]
        Hkc = P.upanel(hu, k)
        M = _gather_m(P, hl, hu, R, C)
        eM, eUkc, eLrk, eUkk, eLkk, eHrk = ext(M), ext(Ukc), ext(Lrk), ext(Ukk), ext(Lkk), ext(Hrk)
        aM, aUkc, aLrk, aUkk, aLkk, aHrk = (np.abs(a) for a in (M, Ukc, Lrk, Ukk, Lkk, Hrk))
        # H(R,K)
        HU = eHrk @ eUkk.T
        steps = [(HU + eM @ eUkc.T, aHrk @ aUkk.T + aM @ aUkc.T, 4 * (ns + nc))]
        # H(K,C), on the stored rows of each column
        stored = np.arange(ns)[:, None] >= (P.ufst[k] - f)[None, :]
        r = eLkk.T @ ext(Hkc) + eLrk.T @ eM
        d = aLkk.T @ np.abs(Hkc) + aLrk.T @ aM
        steps.append((np.where(stored, r, 0), np.where(stored, d, 0), 4 * (ns + m)))
        # H(K,K)
        r = eLkk.T @ ext(Hkk) @ eUkk.T - np.eye(ns) + eLrk.T @ HU
        d = aLkk.T @ np.abs(Hkk) @ aUkk.T + np.eye(ns) + aLrk.T @ (aHrk @ aUkk.T + aM @ aUkc.T)
        steps.append((r, d, 8 * (ns + m)))
        for s, (r, d, c) in enumerate(steps):
            q = ratio(r, d)
            raw[s] = max(raw[s], q)
            scaled[s] = max(scaled[s], q / (c * cf * U))
    return scaled, raw


def _back_blocked(t, b, unit, inv_of, refine):
    """T Z = B for an upper triangle T (unit: its diagonal taken as 1), B's columns the vectors: selinv_trsm_kernel's
    sweep, 16 unknowns at a time from the last block (partial where 16 does not divide ns) up, R = B_j - sum_{p > j} T_jp Z_p, then
    Z_j = inv(T_jj) R with the explicit block inverse inv_of(T_jj), and `refine` steps Z_j += inv (R - T_jj Z_j)"""
    ns = t.shape[0]
    z = b.copy()
    for p0 in range(((ns - 1) // 16) * 16, -1, -16):
        p1 = min(ns, p0 + 16)
        tjj = np.triu(t[p0:p1, p0:p1], 1) + np.eye(p1 - p0) if unit else np.triu(t[p0:p1, p0:p1])
        inv = inv_of(tjj)
        r = z[p0:p1] - t[p0:p1, p1:] @ z[p1:]
        x = inv @ r
        for _ in range(refine):
            x = x + inv @ (r - tjj @ x)
        z[p0:p1] = x
    return z


def selinv_blocked(prob, layer, refine=1):
    """The sweep of slu_selinv.cu in NumPy, on the factors in `layer` -> (hl, hu) as oracle.selinv.selinv returns them.
    Per supernode, the products P = -M U_KC^T, H(K,C) = -L_RK^T M and H(K,K) = I - L_RK^T P, then every row x of
    [H(K,K); P] solves x U_KK^T = x and every column y of [H(K,K) H(K,C)] solves L_KK^T y = y, each by _back_blocked with
    diag_inv_kernel's 16 x 16 inverses (U_bb's, and L_bb's transposed).  refine=0 is the plain product with the inverse,
    refine=1 adds the correction step: for the sensitivity tests of test_selinv_backward_cpu.py only."""
    from oracle.selinv import _Panels
    P = _Panels(prob, layer)
    hl, hu = np.zeros_like(layer.lval), np.zeros_like(layer.uval)
    for k in np.nonzero(layer.held)[0][::-1]:
        ns, Lkk, Ukk, Lrk, Ukc, R, C = _selinv_node(P, layer.lval, layer.uval, k)
        f, klst = int(P.xsup[k]), int(P.xsup[k + 1])
        M = _gather_m(P, hl, hu, R, C)
        Prk = -(M @ Ukc.T)
        Hkc = -(Lrk.T @ M)
        Hkk = np.eye(ns, dtype=hl.dtype) - Lrk.T @ Prk
        rows = _back_blocked(Ukk, np.vstack([Hkk, Prk]).T, False, _inv_upper16, refine).T
        cols = _back_blocked(Lkk.T, np.hstack([rows[:ns], Hkc]), True, lambda t: _inv_unit_lower16(t.T).T, refine)
        Hp = P.lpanel(hl, k)
        Hp[:ns] = cols[:, :ns]
        Hp[ns:] = rows[ns:]
        o = int(layer.uval_off[k])
        for j in range(len(C)):
            fst, seg = int(P.ufst[k][j]), int(P.useg[k][j])
            hu[o + seg:o + seg + klst - fst] = cols[fst - f:, ns + j]
    return hl, hu


def pivot_logdet(prob, layer):
    """(sign or phase, log |det F|, its tolerance, the phase's tolerance) from the pivots of `layer`: log |u_ii| summed
    exactly (math.fsum) and the count of negative pivots, or in complex exp(i theta) with theta = fsum(arg u_ii) mod
    2 pi.  A sum of n correctly rounded terms x_i in any order is within n u sum |x_i| of the exact sum of the terms
    (n - 1 additions, each off by at most u times a partial sum, plus the rounding of each term); a bound in max |x_i|
    alone does not hold for a sequential sum, whose partial sums grow to n max |x_i|."""
    import math
    from oracle.inertia import pivots
    d = pivots(prob, layer)
    logs = np.log(np.abs(d))
    n = len(d)
    la = math.fsum(logs.tolist())
    tol = n * U * float(np.abs(logs).sum())
    if not np.iscomplexobj(d):
        return (-1.0 if np.count_nonzero(d < 0) % 2 else 1.0), la, tol, 0.0
    arg = np.angle(d)
    theta = math.remainder(math.fsum(arg.tolist()), 2 * math.pi)
    return np.exp(1j * theta), la, tol, n * U * (float(np.abs(arg).sum()) + 2 * math.pi)
