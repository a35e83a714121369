"""Iterative refinement costs (slu_b200_gsrfs) against the scaled solve it refines (slu_b200_solve_scaled).

    python scripts/bench_refine.py [--fill-grid G] [--kkt G M] [--reps R]

Prints one JSON line per matrix and nrhs, each with the GPU's name and power limit: solve_scaled alone, gsrfs without the
forward error bound (with its steps and final berr), gsrfs with it (ferr), for nrhs 1 and 8, on the bench.py matrix (fem3
at --fill-grid^3 nodes x 3 dof) and a KKT matrix [K B^T; B 0] (2D Poisson K on G^2, M constraints).  Each gsrfs call starts
from solve_scaled's x.  Times are host wall clock around calls that end in a device synchronise, the median over --reps
after one warm-up call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402
from test_static_pivot_cpu import csr_parts, kkt  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["unknown, unknown"])[0].split(", ")
    return {"gpu": name, "power_limit": power}


def median_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def handle(rp, ci, v, perm_fn):
    n = len(rp) - 1
    perm_r, R, C, _ = hostlib.large_diag_perm(rp, ci, v)
    prp, pci, pv = hostlib.row_permute(rp, ci, v, perm_r)
    perm = perm_fn(perm_r, prp, pci)
    prob = LUProblem.from_matrix(prp, pci, pv, perm, relax=32, maxsup=256)
    h = capi.Handle(prob, 0)
    h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, C)
    assert h.factor() == 0
    return h, n


def measure(h, n, tag, reps, emit):
    rng = np.random.default_rng(0)
    for nrhs in (1, 8):
        b = rng.standard_normal((nrhs, n))
        x0 = h.solve_scaled(b)
        t_solve = median_time(lambda: h.solve_scaled(b), reps)
        _, berr, steps, _ = h.refine(b, x0, ferr=False)
        t_refine = median_time(lambda: h.refine(b, x0, ferr=False), reps)
        launches = int(h.stats().reserved[5])
        _, _, _, ferr = h.refine(b, x0, ferr=True)
        t_ferr = median_time(lambda: h.refine(b, x0, ferr=True), reps)
        launches_ferr = int(h.stats().reserved[5])
        emit(what="refine", nrhs=nrhs, solve_scaled_s=t_solve, gsrfs_s=t_refine, gsrfs_ferr_s=t_ferr,
             steps=[int(s) for s in steps], berr_max=float(berr.max()), ferr_max=float(ferr.max()), launches=launches,
             launches_ferr=launches_ferr, **tag)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fill-grid", type=int, default=40)
    ap.add_argument("--kkt", type=int, nargs=2, default=[200, 10000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    info = gpu_info()

    def emit(**kw):
        print(json.dumps({**kw, **info}), flush=True)

    g = a.fill_grid
    rp, ci, v = hostlib.fem3d(g, g, g, dof=3)
    n = len(rp) - 1
    h, n = handle(rp, ci, v, lambda pr, prp, pci: hostlib.nd_order(g, dof=3, leaf=8) if np.array_equal(pr, np.arange(n))
                  else hostlib.nd_order_graph(prp, pci, leaf=64))
    measure(h, n, dict(matrix=f"fem3-{g}^3x3", n=n, nnz=len(ci)), a.reps, emit)
    h.close()

    rp, ci, v = csr_parts(kkt(a.kkt[0], a.kkt[1], 1))
    h, n = handle(rp, ci, v, lambda pr, prp, pci: hostlib.nd_order_graph(prp, pci, leaf=64))
    measure(h, n, dict(matrix=f"kkt-poisson{a.kkt[0]}^2-{a.kkt[1]}", n=n, nnz=len(ci)), a.reps, emit)
    h.close()


if __name__ == "__main__":
    main()
