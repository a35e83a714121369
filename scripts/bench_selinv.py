"""Selected inversion on the resident factors (slu_b200_selinv, or slu_b200_z_selinv with --dtype c128) against the
factorization and against solves.

    python scripts/bench_selinv.py [--dtype f64|c128] [--workloads poisson fem3] [--poisson-grid 48] [--fem-grid 0]
                                   [--steps K] [--warmup W]

Workloads: Poisson 48^3 with the non-symmetric seeded values of scripts/bench_solve_trans.py, and the FEM workload of
bench.py (27-point, 3 dof per node) at the largest grid whose factors fit twice beside their workspace in 80 GB
(slu_b200_plan sizes them; --fem-grid overrides), with the same kind of values.  Geometric nested dissection, maxsup 256,
relax 64, as bench.py.  Per workload one handle is filled on the device and factored; then, per timed round: factor,
selinv, inv_diag (the diagonal of A^-1) and inv_entries on the pattern of A.  Times: stats.t_factor_s (device events) for
the factorization, the library's host clock around the call (out[0]) for selinv, and a host clock around the Python call
for inv_diag / inv_entries (H2D of the pattern and D2H of the values included); medians over the timed rounds.  TFlop/s =
the library's flop count (out[1]) over the selinv time.  diag(A^-1) by solves: timed batches of 8 unit-vector solves,
extrapolated to n / 8 batches.  Sampled entries of inv_diag are checked against those solves.  Prints one JSON line per
workload with the card's name and power limit read in the same run.  One GPU; writes nothing to disk.
--dtype c128 runs the same on doublecomplex values (bench_solve_trans.values(..., True)); the FEM grid is sized by
slu_b200_z_plan (16 bytes per entry), and the JSON line adds real_tflops = 4 x the library's rate, which counts a complex
multiply-add as 2 flops.
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
from bench_solve_trans import gpu_name_and_power, values  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402

HBM_BYTES = 80e9
FEM_GRIDS = (68, 64, 60, 56, 52, 48, 44, 40, 36)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="f64", choices=["f64", "c128"])
    ap.add_argument("--workloads", nargs="+", default=["poisson", "fem3"], choices=["poisson", "fem3"])
    ap.add_argument("--poisson-grid", type=int, default=48)
    ap.add_argument("--fem-grid", type=int, default=0, help="0: the largest grid of FEM_GRIDS whose factors fit twice")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--solve-batches", type=int, default=4)
    return ap.parse_args()


def symbolic(kind, g):
    a = argparse.Namespace(workload=kind, ordering="geometric", leaf=64)
    rp, ci, v, perm = bench.make_matrix(a, g)
    sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=64, maxsup=256, amalg=0.05)
    return rp, ci, v, sym


def new_problem(sym, cplx):
    prob = LUProblem.from_symbolic(sym, npdep=1)
    if cplx:
        prob.dtype = np.dtype(np.complex128)
    prob.add_layer(0)
    return prob


def fits_twice(sym, cplx):
    prob = new_problem(sym, cplx)
    st = capi.plan(prob, 0)
    return 2 * st.lu_device_bytes + st.index_device_bytes <= 0.9 * HBM_BYTES, st


def run_one(kind, g, rp, ci, v, sym, args, gpu):
    n = len(rp) - 1
    cplx = args.dtype == "c128"
    prob = new_problem(sym, cplx)
    val = values(rp, ci, v, cplx)
    pm = np.asarray(prob.perm, np.int32)
    h = capi.Handle(prob, 0, device=0)
    t_fac, t_si, t_diag, t_ent, out = [], [], [], [], None
    for i in range(args.warmup + args.steps):
        h.fill_csr(rp, ci, val, pm)
        assert h.factor() == 0
        out = h.selinv()
        t0 = time.perf_counter()
        d = h.inv_diag(pm)
        t1 = time.perf_counter()
        e = h.inv_entries(rp, ci, pm)
        t2 = time.perf_counter()
        if i >= args.warmup:
            t_fac.append(h.stats().t_factor_s)
            t_si.append(out[0])
            t_diag.append(t1 - t0)
            t_ent.append(t2 - t1)
    assert np.isfinite(e).all()
    # diag(A^-1) by solves of unit vectors (ordering of the factored matrix: column perm[j] of F^-1 is column j of A^-1)
    rng = np.random.default_rng(2)
    ts, worst = [], 0.0
    for b in range(args.solve_batches + 1):
        cols = rng.choice(n, 8, replace=False)
        rhs = np.zeros((8, n), prob.dtype)
        rhs[np.arange(8), pm[cols]] = 1.0
        x = h.solve(rhs)
        if b:
            ts.append(h.stats().reserved[4])
        ref = x[np.arange(8), pm[cols]]
        worst = max(worst, float(np.max(np.abs(d[cols] - ref) / np.abs(ref))))
    assert worst <= 1e-10, worst
    st = h.stats()
    h.close()
    med = lambda xs: float(np.median(xs))  # noqa: E731
    name = bench.workload_name(g, kind)
    extra = {}
    if cplx:
        name = name.replace("fp64", "c128")
        extra = {"dtype": "c128", "real_tflops": round(4 * out[1] / med(t_si) / 1e12, 2),
                 "flop_count": "library count: a complex multiply-add counts 2, real_tflops = 4 x selinv_tflops"}
    print(bench.json_line({
        "metric": "selinv_ms", "value": round(med(t_si) * 1e3, 2), "unit": "ms", "higher_is_better": False,
        "workload": name, "values": "non-symmetric, diagonally dominant (scripts/bench_solve_trans.py)", "n": n,
        "nnz_lu": int(st.nnz_l + st.nnz_u), "nlevels": int(st.nlevels), "steps": args.steps, "warmup": args.warmup,
        "factor_ms": round(med(t_fac) * 1e3, 2), "selinv_over_factor": round(med(t_si) / med(t_fac), 2),
        "selinv_flops": out[1], "selinv_tflops": round(out[1] / med(t_si) / 1e12, 2), "selinv_launches": int(out[2]),
        "selinv_hbm_bytes": int(out[3]), "inv_diag_ms": round(med(t_diag) * 1e3, 2),
        "inv_entries_pattern_of_A_ms": round(med(t_ent) * 1e3, 2), "nnz_A": len(ci),
        "diag_by_solves_s": round(med(ts) * n / 8, 1), "solve_8rhs_ms": round(med(ts) * 1e3, 2),
        "diag_check_max_rel_err": worst, "gpu": gpu,
        "how": "factor: stats.t_factor_s; selinv: out[0] (host clock around the call); inv_diag / inv_entries: host clock "
               "around the call; diag by solves: n / 8 x the median of timed 8-right-hand-side unit-vector solves", **extra}))


def main():
    args = parse()
    capi.require_gpu()
    gpu = gpu_name_and_power()
    for kind in args.workloads:
        if kind == "poisson":
            g = args.poisson_grid
            rp, ci, v, sym = symbolic(kind, g)
        else:
            for g in ((args.fem_grid,) if args.fem_grid > 0 else FEM_GRIDS):
                rp, ci, v, sym = symbolic(kind, g)
                if args.fem_grid > 0 or fits_twice(sym, args.dtype == "c128")[0]:
                    break
        run_one(kind, g, rp, ci, v, sym, args, gpu)


if __name__ == "__main__":
    main()
