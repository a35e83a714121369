"""Plain, transposed and conjugate-transposed solves on the resident factors of one handle (slu_b200_solve against
slu_b200_solve_trans, and their doublecomplex twins).

    python scripts/bench_solve_trans.py [--grid G] [--nrhs 1 8] [--dtype f64 c128] [--steps K] [--warmup W]

For every dtype and nrhs: one handle of the Poisson G^3 matrix (geometric nested dissection, maxsup 256: the ordering and
supernode settings of bench.py) with non-symmetric, diagonally dominant seeded values is filled on the device and factored
once; then N, T and (complex only) H solves of the same b alternate on it.  Time = stats.reserved[4], the library's host
clock around the call (H2D of b and D2H of x included); median of the timed rounds after the warm-up rounds.  Prints one
JSON line per case with the card's name and power limit and the HBM bound bytes_per_entry * (nnz_l + nnz_u) * nrhs /
3.35 TB/s (one read of L and U per right-hand side at the H100 SXM data-sheet bandwidth).  Every solution of the last
round is checked against its system with SciPy.  One GPU; writes nothing to disk.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=48)
    ap.add_argument("--nrhs", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--dtype", nargs="+", default=["f64", "c128"], choices=["f64", "c128"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--maxsup", type=int, default=256)
    ap.add_argument("--relax", type=int, default=64)
    ap.add_argument("--leaf", type=int, default=64)
    ap.add_argument("--amalg", type=float, default=0.05)
    a = ap.parse_args()
    a.workload, a.ordering = "poisson", "geometric"
    return a


def values(rp, ci, v, cplx, seed=0):
    """Off-diagonal entries scaled by seeded factors in [0.5, 1.5) (plus an imaginary part of up to half their size in
    complex), the diagonal set to the row's off-diagonal 1-norm + 1: non-symmetric, strictly diagonally dominant."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    off = rows != ci
    w = np.where(off, v * rng.uniform(0.5, 1.5, len(v)), 0.0)
    if cplx:
        w = w + 1j * np.where(off, 0.5 * v * rng.uniform(-1.0, 1.0, len(v)), 0.0)
    d = np.bincount(rows, np.abs(w), len(rp) - 1) + 1.0
    return np.where(off, w, d[rows] + (0.25j if cplx else 0.0))


def gpu_name_and_power():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def run(args):
    capi.require_gpu()
    gpu = gpu_name_and_power()
    rp, ci, v, perm = bench.make_matrix(args, args.grid)
    n = len(rp) - 1
    sym = hostlib.Symbolic(n, rp, ci, perm, relax=args.relax, maxsup=args.maxsup, amalg=args.amalg)
    rows = np.repeat(np.arange(n), np.diff(rp))
    for dtype in args.dtype:
        cplx = dtype == "c128"
        prob = LUProblem.from_symbolic(sym, npdep=1)
        if cplx:
            prob.dtype = np.dtype(np.complex128)
        prob.add_layer(0)
        val = values(rp, ci, v, cplx)
        pm = np.asarray(prob.perm)
        F = sp.csr_matrix((val, (pm[rows], pm[ci])), shape=(n, n))      # P A P^T, the ordering of the solves
        ops = {"N": F, "T": F.T.tocsr(), "H": F.conj().T.tocsr()}
        h = capi.Handle(prob, 0, device=0)
        h.fill_csr(rp, ci, val, pm)
        assert h.factor() == 0
        st = h.stats()
        nnz_lu = int(st.nnz_l + st.nnz_u)
        transes = ("N", "T", "H") if cplx else ("N", "T")
        rng = np.random.default_rng(1)
        for nrhs in args.nrhs:
            b = rng.standard_normal((nrhs, n)) + (1j * rng.standard_normal((nrhs, n)) if cplx else 0.0)
            times = {t: [] for t in transes}
            launches, resid = {}, {}
            for i in range(args.warmup + args.steps):
                for t in transes:
                    x = h.solve(b, trans=t)
                    st = h.stats()
                    if i >= args.warmup:
                        times[t].append(st.reserved[4])
                    launches[t] = int(st.reserved[5])
                    if i == args.warmup + args.steps - 1:
                        resid[t] = float(np.linalg.norm(ops[t] @ x.T - b.T) / np.linalg.norm(b))
                        assert resid[t] <= 1e-10, (t, resid[t])
            med = {t: float(np.median(times[t])) for t in transes}
            bound_s = 8 * (2 if cplx else 1) * nnz_lu * nrhs / HBM_BYTES_PER_S
            print(bench.json_line({
                "metric": "solve_trans_ms", "value": round(med["T"] * 1e3, 3), "unit": "ms", "higher_is_better": False,
                "dtype": dtype, "nrhs": nrhs, "workload": bench.workload_name(args.grid).replace("fp64", dtype),
                "n": n, "nnz_lu": nnz_lu, "steps": args.steps, "warmup": args.warmup,
                "solve_ms": {t: round(med[t] * 1e3, 3) for t in transes},
                "ratio_to_N": {t: round(med[t] / med["N"], 3) for t in transes},
                "hbm_bound_ms": round(bound_s * 1e3, 3), "launches": launches, "residual": resid, "gpu": gpu,
                "how": "stats.reserved[4] (host clock around the call, H2D of b and D2H of x included), N/T/H alternating "
                       "on one handle, median of the timed rounds"}))
        h.close()


if __name__ == "__main__":
    run(parse())
