"""oracle/inertia.py, the NumPy restatement of slu_b200_inertia, on the oracle's factors: eigenvalue counts of A - sigma I
against the analytic 7-point spectrum, of a pencil (K, M) against scipy.linalg.eigh(K, M), of a complex Hermitian matrix
with random flux against eigvalsh, and the tiny-pivot count against the oracle's own.  The shifts chosen here are the ones
the GPU tests (test_gpu_inertia.py) reuse: all are dyadic, so that K - sigma M is exact in both routes, and each lies well
inside a gap of the spectrum.  An unpivoted indefinite factorization can lose a count near an eigenvalue of a leading
block; a shift that did so would be a bad test input, and these tests show that none of these does."""
import numpy as np
import pytest
import scipy.linalg as sla

from oracle import inertia, oracle
from test_scaled_parity import make_problem
from util import load_fixture, poisson_problem

SMALL = [dict(N=8, leaf=4, relax=8, maxsup=32), dict(N=10, leaf=8, relax=16, maxsup=128)]
# Poisson 32^3 (ND, leaf 16), the GPU scale test: shifts among the lowest 400 eigenvalues, checked below with the oracle
BIG = dict(N=32, leaf=16, relax=32, maxsup=256)
BIG_WIDE = dict(N=32, leaf=16, relax=32, maxsup=512)
SHIFTS32 = [0.041015625, 0.103515625, 0.20703125, 0.3955078125, 0.84765625]
# the defect of a Hermitian input: rounding in Im u_ii relative to |u_ii|, which an indefinite shift can make small (up to
# 3e-10 on the oracle's factors of the flux matrices here, 5e-8 on the GPU's; 0 on real factors)
DEFECT_TOL = 1e-6
# shifts of the tiny-pivot fixture's diagonal whose factorizations replace pivots (no pivot lands on thresh by cancellation)
TINY_SHIFTS = [0.0, 4.0, 5.0]


def spectrum(N):
    """The eigenvalues of hostlib.poisson3d(N) (diagonal 6, off-diagonal -1, Dirichlet): sum_d 4 sin^2(k_d pi / 2(N + 1))"""
    k = np.arange(1, N + 1)
    l1 = 4.0 * np.sin(k * np.pi / (2 * (N + 1))) ** 2
    return np.sort((l1[:, None, None] + l1[None, :, None] + l1[None, None, :]).ravel())


def gap_shifts(ev, count, scale=64, margin=1e-3):
    """`count` shifts spread over the spectrum ev: multiples of 1 / scale, each more than `margin` from every eigenvalue.
    No integers: the leading blocks of the 7-point Laplacian have many integer eigenvalues (6, its diagonal, among them),
    where the unpivoted factorization meets exact zero pivots."""
    d = np.unique(np.round(ev, 10))
    s = np.round((d[:-1] + d[1:]) / 2 * scale) / scale
    ok = (s - d[:-1] > margin) & (d[1:] - s > margin) & (s != np.round(s))
    s = s[ok]
    return [float(x) for x in s[np.linspace(0, len(s) - 1, count).round().astype(int)]]


def rows_of(rp):
    return np.repeat(np.arange(len(rp) - 1), np.diff(rp))


def shifted(rp, ci, v, sigma, m=None):
    """K - sigma M on the CSR values (M = I when m is None)"""
    if m is None:
        return np.where(rows_of(rp) == np.asarray(ci), v - sigma, v)
    return v - sigma * m


def mass_values(rp, ci):
    """An SPD M on the pattern: diagonal 1, off-diagonal 1/8 (at most 6 neighbours: diagonally dominant)"""
    return np.where(rows_of(rp) == np.asarray(ci), 1.0, 0.125)


def flux_values(rp, ci, v, seed=0):
    """A complex Hermitian matrix on the pattern of the real symmetric v: a_ij = v_ij e^{i theta_ij}, theta_ji = -theta_ij
    random (a magnetic Laplacian with random flux)"""
    rows, ci = rows_of(rp), np.asarray(ci)
    n = len(rp) - 1
    lo, hi = np.minimum(rows, ci), np.maximum(rows, ci)
    theta = np.random.default_rng(seed).uniform(-np.pi, np.pi, n * n)[lo * n + hi]   # one angle per edge
    return v * np.exp(1j * np.where(rows < ci, theta, np.where(rows > ci, -theta, 0.0)))


def dense(rp, ci, vals):
    n = len(rp) - 1
    A = np.zeros((n, n), np.asarray(vals).dtype)
    A[rows_of(rp), ci] = vals
    return A


def counts_of(kw, vals):
    prob = make_problem(kw, vals)
    info, _, tiny = oracle.factor(prob)
    assert info == 0
    neg, pos, tn, defect = inertia.inertia(prob, prob.layers[0])
    assert neg + pos == prob.n and tn == tiny
    return neg, tn, defect


@pytest.mark.parametrize("kw", SMALL, ids=["poisson8", "poisson10"])
def test_shifted_laplacian_against_analytic_spectrum(kw):
    _, (rp, ci, v) = poisson_problem(**kw)
    ev = spectrum(kw["N"])
    assert np.abs(ev - np.linalg.eigvalsh(dense(rp, ci, v))).max() < 1e-12
    for s in gap_shifts(ev, 7):
        neg, tiny, defect = counts_of(kw, shifted(rp, ci, v, s))
        assert (neg, tiny, defect) == (int(np.sum(ev < s)), 0, 0.0), s


@pytest.mark.parametrize("kw", SMALL, ids=["poisson8", "poisson10"])
def test_pencil_against_eigh(kw):
    _, (rp, ci, v) = poisson_problem(**kw)
    m = mass_values(rp, ci)
    ev = sla.eigh(dense(rp, ci, v), dense(rp, ci, m), eigvals_only=True)
    for s in gap_shifts(ev, 5):
        assert counts_of(kw, shifted(rp, ci, v, s, m)) == (int(np.sum(ev < s)), 0, 0.0), s


@pytest.mark.parametrize("kw", SMALL, ids=["poisson8", "poisson10"])
def test_hermitian_flux_against_eigvalsh(kw):
    _, (rp, ci, v) = poisson_problem(**kw)
    a = flux_values(rp, ci, v, seed=kw["N"])
    A = dense(rp, ci, a)
    assert np.abs(A - A.conj().T).max() == 0.0
    ev = np.linalg.eigvalsh(A)
    for s in gap_shifts(ev, 5):
        neg, tiny, defect = counts_of(kw, shifted(rp, ci, a, s))
        assert neg == int(np.sum(ev < s)) and tiny == 0 and defect <= DEFECT_TOL, (s, neg, defect)


def test_non_hermitian_complex_defect_is_large():
    kw = SMALL[0]
    _, (rp, ci, v) = poisson_problem(**kw)
    a = shifted(rp, ci, v, 0.5) + 0j
    a[rows_of(rp) == np.asarray(ci)] += 0.25j            # A - (0.5 - 0.25 i) I: complex symmetric, not Hermitian
    _, _, defect = counts_of(kw, a)
    assert defect > 1e-3


def diag_positions(prob, lay):
    """lval indices of the diagonal of F in the diagonal blocks"""
    xsup = np.asarray(prob.xsup, np.int64)
    out = []
    for k in np.nonzero(lay.held)[0]:
        ns, nsupr = int(xsup[k + 1] - xsup[k]), int(prob.lidx[prob.lidx_off[k] + 1])
        out.append(int(lay.lval_off[k]) + np.arange(ns) * (nsupr + 1))
    return np.concatenate(out)


@pytest.mark.parametrize("sigma", TINY_SHIFTS)
def test_tiny_count_equals_oracle_replacements(sigma):
    """poisson12_nd_tiny (replacement on) with sigma subtracted from the diagonal of F: every replaced pivot is +-thresh,
    and the restatement's count of |u_ii| <= thresh equals the oracle's count of replacements"""
    prob, _, _ = load_fixture("poisson12_nd_tiny")
    lay = prob.layers[0]
    assert prob.replace_tiny_pivot and prob.thresh > 0
    lay.lval[diag_positions(prob, lay)] -= sigma
    info, _, tiny = oracle.factor(prob)
    neg, pos, tn, _ = inertia.inertia(prob, lay)
    assert info == 0 and tn == tiny and neg + pos == prob.n
    if sigma:
        assert tiny > 0
    else:
        assert (neg, tiny) == (0, 0)


@pytest.mark.parametrize("kw", [BIG, BIG_WIDE], ids=["w256", "w512"])
def test_poisson32_shifts_against_analytic_spectrum(kw):
    """The 32^3 shifts of the GPU scale test: the oracle's unpivoted factorization gives the analytic counts"""
    _, (rp, ci, v) = poisson_problem(**kw)
    ev = spectrum(32)
    for s in SHIFTS32:
        assert np.min(np.abs(ev - s)) > 1e-3 and np.sum(ev < s) < 400
        assert counts_of(kw, shifted(rp, ci, v, s)) == (int(np.sum(ev < s)), 0, 0.0), s
