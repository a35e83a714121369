"""Static pivoting costs (slu_b200_fill_csr_scaled / _solve_scaled and the host matching sluh_large_diag_perm).

    python scripts/bench_scaled.py [--fill-grid G] [--kkt G M] [--reps R]

Prints one JSON line per measurement, each with the GPU's name and power limit:
  * sluh_large_diag_perm on the bench.py matrix (fem3, 68^3 nodes x 3 dof: n = 943,296) and on a KKT matrix
    [K B^T; B 0] (2D Poisson K on G^2, M constraints);
  * fill_csr_scaled with and without the device equilibration against fill_csr of the same values (fem3 at --fill-grid);
  * solve_scaled against solve plus the NumPy permute and scale of b and x around it (nrhs 1).
Times are host wall clock around calls that end in a device synchronise, the median over --reps after one warm-up call.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fill-grid", type=int, default=40)
    ap.add_argument("--kkt", type=int, nargs=2, default=[400, 40000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    info = gpu_info()

    def emit(**kw):
        print(json.dumps({**kw, **info}), flush=True)

    rp, ci, v = hostlib.fem3d(68, 68, 68, dof=3)
    t0 = time.perf_counter()
    hostlib.large_diag_perm(rp, ci, v)
    emit(what="sluh_large_diag_perm", matrix="fem3-68^3x3", n=len(rp) - 1, nnz=len(ci), seconds=time.perf_counter() - t0)
    del rp, ci, v
    rp, ci, v = csr_parts(kkt(a.kkt[0], a.kkt[1], 1))
    t0 = time.perf_counter()
    hostlib.large_diag_perm(rp, ci, v)
    emit(what="sluh_large_diag_perm", matrix=f"kkt-poisson{a.kkt[0]}^2-{a.kkt[1]}", n=len(rp) - 1, nnz=len(ci),
         seconds=time.perf_counter() - t0)

    g = a.fill_grid
    rp, ci, v = hostlib.fem3d(g, g, g, dof=3)
    n = len(rp) - 1
    perm_r, R, C, _ = hostlib.large_diag_perm(rp, ci, v)
    prp, pci, pv = hostlib.row_permute(rp, ci, v, perm_r)
    perm = hostlib.nd_order(g, dof=3, leaf=8) if np.array_equal(perm_r, np.arange(n)) else hostlib.nd_order_graph(prp, pci, leaf=64)
    prob = LUProblem.from_matrix(prp, pci, pv, perm, relax=32, maxsup=256)
    h = capi.Handle(prob, 0)
    rows = np.repeat(np.arange(n), np.diff(rp))
    sv = (v * R[rows]) * C[ci]
    srp, sci, ssv = hostlib.row_permute(rp, ci, sv, perm_r)
    tag = dict(matrix=f"fem3-{g}^3x3", n=n, nnz=len(ci))
    t_plain = median_time(lambda: h.fill_csr(srp, sci, ssv, prob.perm), a.reps)
    t_scaled = median_time(lambda: h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, C, equil=False), a.reps)
    t_equil = median_time(lambda: h.fill_csr_scaled(rp, ci, v, prob.perm, perm_r, R, C, equil=True), a.reps)
    emit(what="fill", fill_csr_s=t_plain, fill_csr_scaled_s=t_scaled, fill_csr_scaled_equil_s=t_equil, **tag)

    assert h.factor() == 0
    _, Rf, Cf = h.scaling()
    rmap = prob.perm[perm_r]
    b = np.random.default_rng(0).standard_normal(n)

    def numpy_around_solve():
        bp = np.empty(n)
        bp[rmap] = Rf * b
        y = h.solve(bp)
        return Cf * y[prob.perm]

    x1 = h.solve_scaled(b)
    x2 = numpy_around_solve()
    assert np.abs(x1 - x2).max() <= 1e-12 * np.abs(x2).max()
    t_s = median_time(lambda: h.solve_scaled(b), a.reps)
    launches = int(h.stats().reserved[5])
    t_n = median_time(numpy_around_solve, a.reps)
    emit(what="solve", solve_scaled_s=t_s, solve_plus_numpy_s=t_n, launches_scaled=launches, **tag)
    h.close()


if __name__ == "__main__":
    main()
