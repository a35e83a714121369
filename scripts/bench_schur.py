"""Partial factorization with a Schur complement (capi.SchurHandle: slu_b200_schur_*) against the full factorization of
the same matrix.

    python scripts/bench_schur.py [--workloads poisson fem3] [--poisson-grid 48] [--fem-grid 68] [--steps K] [--warmup W]

Workloads: Poisson 48^3 and the FEM workload of bench.py (27-point, 3 dof per node, 68^3 nodes by default), with the
non-symmetric, diagonally dominant values of scripts/bench_solve_trans.py.  Geometric nested dissection, maxsup 256,
relax 64, as bench.py; the Schur set is the top-level separator of that ordering (a plane of g^2 nodes: s = g^2 x dof),
which sluh_symbolic_schur keeps last.  Both arms use this one symbolic structure: the full arm is an ordinary handle that
factors every supernode, the partial arm a Schur handle.  Per timed round: fill_csr + factor in each arm; schur_get,
condense + expand on the partial handle; one solve on the full one.  Times: stats.t_factor_s (device events) for the
factorizations, stats.reserved[6] (host clock around the call: memset, gather, D2H of s x s into pageable memory) and
stats.reserved[7] (device events around the gather kernel) for schur_get, stats.reserved[4] for condense, expand and the
solve (H2D of b and D2H of x included); medians over the timed rounds.  The gather's byte bound is (stored entries of the
Schur panels + s^2) x 8 bytes over 3.35 TB/s.  The composed solve x2 = S^-1 g (a dense LU of S on the GPU through torch,
outside the library) is checked by its residual ||A x - b|| / (||A|| ||x|| + ||b||).  Prints one JSON line per workload
with the card's name and power limit read in the same run.  One GPU; writes nothing to disk.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
from bench_solve_trans import gpu_name_and_power, values  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402

HBM_BW = 3.35e12     # H100 SXM HBM3, data sheet


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["poisson", "fem3"], choices=["poisson", "fem3"])
    ap.add_argument("--poisson-grid", type=int, default=48)
    ap.add_argument("--fem-grid", type=int, default=68)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    return ap.parse_args()


def problem(kind, g):
    a = argparse.Namespace(workload=kind, ordering="geometric", leaf=64)
    rp, ci, v, perm = bench.make_matrix(a, g)
    s = g * g * (3 if kind == "fem3" else 1)
    sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=64, maxsup=256, amalg=0.05, nschur=s)
    prob = LUProblem.from_symbolic(sym, npdep=1)
    prob.add_layer(0)
    return rp, ci, v, prob, s


def stored_schur_entries(prob, s):
    xsup = np.asarray(prob.xsup)
    k1 = int(np.searchsorted(xsup, prob.n - s))
    return int(np.asarray(prob.lval_len)[k1:].sum() + np.asarray(prob.uval_len)[k1:].sum())


def run_one(kind, g, args, gpu):
    import scipy.sparse as sp
    import torch
    rp, ci, v, prob, s = problem(kind, g)
    n, n1 = prob.n, prob.n - s
    val = values(rp, ci, v, False)
    pm = np.asarray(prob.perm, np.int32)
    med = lambda xs: float(np.median(xs))  # noqa: E731
    b = np.random.default_rng(4).standard_normal(n)

    # full factorization of the same structure, then one solve
    h = capi.Handle(prob, 0, device=0)
    t_full, t_solve = [], []
    for i in range(args.warmup + args.steps):
        h.fill_csr(rp, ci, val, pm)
        assert h.factor() == 0
        h.solve(b)
        if i >= args.warmup:
            t_full.append(h.stats().t_factor_s)
            t_solve.append(h.stats().reserved[4])
    sf = h.stats()
    h.close()

    # partial factorization
    h = capi.SchurHandle(prob, s, device=0)
    t_part, t_get, t_gather, t_cond, t_exp = [], [], [], [], []
    for i in range(args.warmup + args.steps):
        h.fill_csr(rp, ci, val, pm)
        assert h.factor() == 0
        S = h.schur()
        y = h.condense(b)
        tc = h.stats().reserved[4]
        st = h.stats()
        yy = y.copy()
        yy[n1:] = 0.0
        h.expand(yy)
        if i >= args.warmup:
            t_part.append(st.t_factor_s)
            t_get.append(st.reserved[6])
            t_gather.append(st.reserved[7] * 1e-3)
            t_cond.append(tc)
            t_exp.append(h.stats().reserved[4])
    sp_ = h.stats()
    St = torch.from_numpy(S).cuda()
    x2 = torch.linalg.solve(St, torch.from_numpy(y[n1:]).cuda()).cpu().numpy()
    del St
    torch.cuda.empty_cache()
    y[n1:] = x2
    x = h.expand(y)
    h.close()
    A = sp.csr_matrix((val, ci, rp), shape=(n, n))
    xo = x[pm]                                       # original ordering: x_orig[i] = x_F[perm[i]]
    bo = b[pm]
    res = float(np.linalg.norm(A @ xo - bo) / (sp.linalg.norm(A, np.inf) * np.linalg.norm(xo) + np.linalg.norm(bo)))
    stored = stored_schur_entries(prob, s)
    bound = (stored + s * s) * 8.0 / HBM_BW
    print(bench.json_line({
        "metric": "schur_factor_ms", "value": round(med(t_part) * 1e3, 2), "unit": "ms", "higher_is_better": False,
        "workload": bench.workload_name(g, kind), "schur_set": "top-level separator of the geometric ND", "n": n, "s": s,
        "values": "non-symmetric, diagonally dominant (scripts/bench_solve_trans.py)", "steps": args.steps,
        "warmup": args.warmup, "full_factor_ms": round(med(t_full) * 1e3, 2),
        "partial_over_full": round(med(t_part) / med(t_full), 3),
        "nlevels_full": int(sf.nlevels), "nlevels_partial": int(sp_.nlevels),
        "launches_full": int(sf.gpu_launches), "launches_partial": int(sp_.gpu_launches),
        "ops_full": sf.ops_fact, "ops_partial": sp_.ops_fact,
        "schur_get_ms": round(med(t_get) * 1e3, 2), "gather_kernel_ms": round(med(t_gather) * 1e3, 3),
        "gather_byte_bound_ms": round(bound * 1e3, 3), "gather_share_of_bound": round(bound / med(t_gather), 3),
        "schur_stored_entries": stored, "schur_bytes": s * s * 8,
        "condense_ms": round(med(t_cond) * 1e3, 2), "expand_ms": round(med(t_exp) * 1e3, 2),
        "full_solve_ms": round(med(t_solve) * 1e3, 2), "composed_solve_residual": res, "gpu": gpu,
        "how": "factor: stats.t_factor_s; schur_get: stats.reserved[6] (host clock, D2H included); gather: stats.reserved[7] "
               "(device events); condense / expand / solve: stats.reserved[4] (host clock, transfers included); medians"}))


def main():
    args = parse()
    capi.require_gpu()
    gpu = gpu_name_and_power()
    for kind in args.workloads:
        run_one(kind, args.poisson_grid if kind == "poisson" else args.fem_grid, args, gpu)


if __name__ == "__main__":
    main()
