"""Batched factorization and solve (slu_b200_batch_*) against a sequential loop of one unbatched handle.

    python scripts/bench_batch.py --batch B [--dtype f64|c128] [--workload poisson|fem3] [--grid G] [--steps K] [--warmup W]

B matrices with the pattern of the bench.py workload at --grid (seeded values, matgen.batch_values) are factored and
solved (nrhs = 1) on ONE batched handle, and the same B factorizations and solves are done one member after another on
one unbatched handle.  Prints one JSON line (metric batched_factor_ms_per_member) with both times per member, the
aggregate GFlop/s, the launch counts of both arms and the maximum residual probe over the members.  One GPU; writes
nothing to disk.

--dtype c128 runs the doublecomplex handles (slu_b200_z_batch_* against slu_b200_z_*) on frequency-sweep-like members:
the workload's matrix with i * 0.5 * its diagonal added, then the same seeded scaling.  Their Hermitian part is the
symmetric part of the real matrix (diagonally dominant, positive diagonal: positive definite), so every member has an
unpivoted LU.  The residual probe is real-only; in its place the line reports the maximum over the members of the
relative residual ||A_j x_j - b_j|| / ||b_j|| of the batched solve (scipy.sparse, ordering of the factored matrix).
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib, matgen  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, required=True, help="members B >= 1")
    ap.add_argument("--dtype", default="f64", choices=["f64", "c128"])
    ap.add_argument("--workload", default="poisson", choices=["poisson", "fem3"])
    ap.add_argument("--grid", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--maxsup", type=int, default=256)
    ap.add_argument("--relax", type=int, default=64)
    ap.add_argument("--leaf", type=int, default=64)
    ap.add_argument("--ordering", choices=["geometric", "graph"], default="geometric")
    ap.add_argument("--amalg", type=float, default=0.05)
    ap.add_argument("--no-lookahead", type=int, default=0)
    a = ap.parse_args()
    if a.batch < 1:
        ap.error("--batch must be >= 1")
    return a


def run(args):
    """B members of the workload's pattern on one batched handle vs one unbatched handle looping over them.
    Factor times are device times of the library's factor call (stats.t_factor_s, CUDA events): the batched call once,
    the sequential loop summed over the members; solve times are the library's host clock around its solve call (H2D of b
    and D2H of x included, stats.reserved[4]), nrhs = 1.  Median over the timed steps, after the warm-up steps.  Both
    arms run the FP64 DMMA kernels (the int8 path is off in the unbatched arm, as batched handles never take it)."""
    capi.require_gpu()
    nb, G = args.batch, args.grid
    cplx = args.dtype == "c128"
    rp, ci, v, perm = bench.make_matrix(args, G)
    sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=args.relax, maxsup=args.maxsup, amalg=args.amalg)
    prob = LUProblem.from_symbolic(sym, npdep=1)
    del sym
    if cplx:
        prob.dtype = np.dtype(np.complex128)
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        v = v + 1j * np.where(rows == ci, 0.5 * v, 0.0)      # K + i w C with C = 0.5 diag(K)
    lay = prob.add_layer(0)
    vals = matgen.batch_values(rp, ci, v, nb, seed=0)
    pm = np.asarray(prob.perm)
    n, every = prob.n, np.ones(prob.nsupers, bool)
    # b_j = A_j x in the ordering of the factored matrix, x = +-1 (the reference's xtrue pattern)
    xt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    if cplx:
        import scipy.sparse as sp
        member = lambda j: sp.csr_matrix((vals[j], (pm[rows], pm[ci])), shape=(n, n))   # P A_j P^T
        b = np.stack([member(j) @ xt for j in range(nb)])
    else:
        b = np.empty((nb, n))
        for j in range(nb):
            prob.fill_layer(0, rp, ci, vals[j])
            b[j] = prob.matvec([(lay, every)], xt, 0)
    opt = dict(device=0, schur_variant=0, no_lookahead=args.no_lookahead)

    def median(xs):
        return float(np.median(xs))

    # batched arm
    bh = capi.BatchHandle(prob, nb, **opt)
    tb, sb = [], []
    for i in range(args.warmup + args.steps):
        bh.fill_csr(rp, ci, vals, pm)
        info = bh.factor()
        assert not info.any(), info
        x = bh.solve(b)
        st = bh.stats()
        if i >= args.warmup:
            tb.append(st.t_factor_s)
            sb.append(st.reserved[4])
    solve_err = float(np.abs(x - xt).max())
    assert solve_err < 1e-8, solve_err
    launches_b, solve_launches_b = int(st.gpu_launches), int(st.reserved[5])
    ops_total = float(st.ops_fact)
    nnz_lu = int(st.nnz_l + st.nnz_u) // nb
    if cplx:      # what the timed path computed: every member's solution against its matrix
        resid = max(float(np.linalg.norm(member(j) @ x[j] - b[j]) / np.linalg.norm(b[j])) for j in range(nb))
        assert resid <= 1e-10, f"relative residual {resid} exceeds 1e-10"
    else:         # what the timed path computed: every member's factors against its matrix (residual probe, +-1 vectors)
        rng = np.random.default_rng(0)
        xp = rng.choice([-1.0, 1.0], size=(2, n))
        resid = 0.0
        for j in range(nb):
            bh.download(j)
            yl = prob.matvec([(lay, every)], prob.matvec([(lay, every)], xp, 2), 3)
            prob.fill_layer(0, rp, ci, vals[j])
            ya = prob.matvec([(lay, every)], xp, 0)
            resid = max(resid, float(np.linalg.norm(yl - ya) / np.linalg.norm(ya)))
        assert resid < 1e-10, f"residual probe {resid} exceeds 1e-10"
    bh.close()

    # sequential arm: one unbatched handle, member after member
    h = capi.Handle(prob, 0, tc_slices=-1, **opt)
    ts, ss = [], []
    for i in range(args.warmup + args.steps):
        tf = tsv = 0.0
        for j in range(nb):
            h.fill_csr(rp, ci, vals[j], pm)
            assert h.factor() == 0
            tf += h.stats().t_factor_s
            xj = h.solve(b[j])
            tsv += h.stats().reserved[4]
        if i >= args.warmup:
            ts.append(tf)
            ss.append(tsv)
    assert np.abs(xj - xt).max() < 1e-8
    st1 = h.stats()
    launches_1, solve_launches_1 = int(st1.gpu_launches), int(st1.reserved[5])
    h.close()

    t_b, t_s, s_b, s_s = median(tb), median(ts), median(sb), median(ss)
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = None
    workload = bench.workload_name(G, args.workload, args.ordering)
    print(bench.json_line({
        "metric": "batched_factor_ms_per_member", "value": round(t_b / nb * 1e3, 4), "unit": "ms", "higher_is_better": False,
        "batch": nb, "members": nb, "steps": args.steps, "warmup": args.warmup, "dtype": args.dtype, "data": "synthetic",
        "workload": workload.replace("fp64", "c128") if cplx else workload, "n": n, "nnz_lu_per_member": nnz_lu,
        "factor": {"batched_ms": round(t_b * 1e3, 4), "sequential_ms": round(t_s * 1e3, 4),
                   "batched_ms_per_member": round(t_b / nb * 1e3, 4), "sequential_ms_per_member": round(t_s / nb * 1e3, 4),
                   "speedup_per_member": round(t_s / t_b, 3), "gflops_batched": round(ops_total / t_b * 1e-9, 2),
                   "gflops_sequential": round(ops_total / t_s * 1e-9, 2)},
        "solve_nrhs1": {"batched_ms": round(s_b * 1e3, 4), "sequential_ms": round(s_s * 1e3, 4),
                        "batched_ms_per_member": round(s_b / nb * 1e3, 4), "sequential_ms_per_member": round(s_s / nb * 1e3, 4),
                        "speedup_per_member": round(s_s / s_b, 3), "solve_error_inf": solve_err},
        "gpu_launches": {"batched_factor": launches_b, "unbatched_factor": launches_1,
                         "batched_solve": solve_launches_b, "unbatched_solve": solve_launches_1},
        ("residual" if cplx else "residual_probe"): resid, "gpu": gpu,
        "how": "factor: stats.t_factor_s (device time; sequential = sum over the members); solve: stats.reserved[4] (host "
               "clock, H2D of b and D2H of x included); median of the timed steps"}))


if __name__ == "__main__":
    run(parse())
