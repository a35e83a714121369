"""Condition estimation on the resident factors (slu_b200_gscon, slu_b200_z_gscon, slu_b200_batch_gscon and
slu_b200_z_batch_gscon), against the solves it is made of.

    python scripts/bench_gscon.py [--grid G] [--dtype f64 c128] [--batch-cases poisson:16 poisson:32 fem3:12]
                                  [--batch 1 8 64] [--steps K] [--warmup W]

Part 1, one handle: the Poisson G^3 matrix of scripts/bench_solve_trans.py (geometric nested dissection, maxsup 256,
non-symmetric diagonally dominant seeded values), factored once; then gscon (norm '1') and a plain solve of nrhs 1
alternate.  gscon time = stats.reserved[6], rounds = stats.reserved[7]; solve time = stats.reserved[4] (host clocks around
the calls, with their synchronisations; the solve includes the H2D of b and D2H of x, gscon moves no vector).  The line
reports the median gscon time and the median solve time times the rounds.

Part 2, batched: for every workload and B, B members (matgen.batch_values of the workload, seed 0) on one batched handle,
one batch_gscon call, against one unbatched handle that is filled and factored with each member in turn and runs gscon on
it (only the gscon calls are timed).  Both as milliseconds per member, median over the timed steps.  Every batched rcond
is checked against the unbatched one.

Prints one JSON line per case with the card's name and power limit.  One GPU; writes nothing to disk.
"""
import argparse
import os
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
from bench_solve_trans import gpu_name_and_power, values  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib, matgen  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=48)
    ap.add_argument("--dtype", nargs="+", default=["f64", "c128"], choices=["f64", "c128"])
    ap.add_argument("--batch-cases", nargs="+", default=["poisson:16", "poisson:32", "fem3:12"])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--maxsup", type=int, default=256)
    ap.add_argument("--relax", type=int, default=64)
    ap.add_argument("--leaf", type=int, default=64)
    ap.add_argument("--amalg", type=float, default=0.05)
    a = ap.parse_args()
    a.ordering = "geometric"
    return a


def anorm1(rp, ci, val):
    n = len(rp) - 1
    return float(np.abs(sp.csr_matrix((val, ci, rp), shape=(n, n))).sum(axis=0).max())


def problem(args, workload, grid, cplx):
    args.workload = workload
    rp, ci, v, perm = bench.make_matrix(args, grid)
    sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=args.relax, maxsup=args.maxsup, amalg=args.amalg)
    prob = LUProblem.from_symbolic(sym, npdep=1)
    if cplx:
        prob.dtype = np.dtype(np.complex128)
    prob.add_layer(0)
    return prob, rp, ci, v


def single(args, gpu):
    for dtype in args.dtype:
        cplx = dtype == "c128"
        prob, rp, ci, v = problem(args, "poisson", args.grid, cplx)
        val = values(rp, ci, v, cplx)
        anorm = anorm1(rp, ci, val)
        h = capi.Handle(prob, 0, device=0)
        h.fill_csr(rp, ci, val, prob.perm)
        assert h.factor() == 0
        b = np.ones(prob.n, prob.dtype)
        tg, ts, rounds, rc = [], [], set(), None
        for i in range(args.warmup + args.steps):
            rc = h.rcond(anorm, "1")
            st = h.stats()
            rounds.add(int(st.reserved[7]))
            tg_i = st.reserved[6]
            h.solve(b)
            if i >= args.warmup:
                tg.append(tg_i)
                ts.append(h.stats().reserved[4])
        h.close()
        assert len(rounds) == 1 and 0 < rc <= 1, (rounds, rc)
        r = rounds.pop()
        med_g, med_s = float(np.median(tg)), float(np.median(ts))
        print(bench.json_line({
            "metric": "gscon_ms", "value": round(med_g * 1e3, 3), "unit": "ms", "higher_is_better": False,
            "dtype": dtype, "workload": bench.workload_name(args.grid).replace("fp64", dtype), "n": prob.n,
            "rounds": r, "solve_ms": round(med_s * 1e3, 3), "rounds_x_solve_ms": round(r * med_s * 1e3, 3),
            "ratio_to_rounds_x_solve": round(med_g / (r * med_s), 3), "rcond": rc, "steps": args.steps, "warmup": args.warmup,
            "gpu": gpu, "how": "stats.reserved[6] and [4] (host clocks around the calls), gscon and solve alternating on "
                              "one handle, medians of the timed rounds"}))


def batched(args, gpu):
    for case in args.batch_cases:
        workload, grid = case.split(":")
        grid = int(grid)
        prob, rp, ci, v = problem(args, workload, grid, False)
        for nb in args.batch:
            vals = matgen.batch_values(rp, ci, v, nb, seed=0)
            anorm = np.array([anorm1(rp, ci, vals[j]) for j in range(nb)])
            bh = capi.BatchHandle(prob, nb, device=0)
            bh.fill_csr(rp, ci, vals, prob.perm)
            assert not bh.factor().any()
            tb = []
            for i in range(args.warmup + args.steps):
                rcb = bh.rcond(anorm, "1")
                if i >= args.warmup:
                    tb.append(bh.stats().reserved[6] / nb)
            rounds_b = int(bh.stats().reserved[7])
            bh.close()
            h = capi.Handle(prob, 0, device=0, tc_slices=-1)
            ts, rcs, rounds_s = [], np.zeros(nb), 0
            for i in range(args.warmup + args.steps):
                t = 0.0
                for j in range(nb):
                    h.fill_csr(rp, ci, vals[j], prob.perm)
                    assert h.factor() == 0
                    rcs[j] = h.rcond(anorm[j], "1")
                    st = h.stats()
                    t += st.reserved[6]
                    rounds_s = max(rounds_s, int(st.reserved[7]))
                if i >= args.warmup:
                    ts.append(t / nb)
            h.close()
            err = float(np.abs(rcb - rcs).max() / np.abs(rcs).max())
            assert err <= 1e-10, err
            mb, ms = float(np.median(tb)), float(np.median(ts))
            print(bench.json_line({
                "metric": "batch_gscon_ms_per_member", "value": round(mb * 1e3, 4), "unit": "ms", "higher_is_better": False,
                "workload": bench.workload_name(grid, workload), "n": prob.n, "batch": nb,
                "sequential_ms_per_member": round(ms * 1e3, 4), "speedup": round(ms / mb, 2),
                "rounds_batched": rounds_b, "max_rounds_sequential": rounds_s, "rcond_rel_diff": err,
                "steps": args.steps, "warmup": args.warmup, "gpu": gpu,
                "how": "stats.reserved[6]: one batch_gscon call / B against the sum of B unbatched gscon calls / B, medians"}))


if __name__ == "__main__":
    a = parse()
    capi.require_gpu()
    g = gpu_name_and_power()
    single(a, g)
    batched(a, g)
