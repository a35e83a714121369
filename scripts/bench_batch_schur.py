"""Partial factorization on a batched handle (capi.BatchSchurHandle: slu_b200_batch_schur_*) against one unbatched
Schur handle (capi.SchurHandle) looping over the members.

    python scripts/bench_batch_schur.py [--workloads p16_faces p12_faces fem18_top] [--batch B ...] [--dtype f64|c128]
                                        [--steps K] [--warmup W]

Workloads (B by default):
  p16_faces   Poisson 16^3 (7-point), the six boundary faces as the Schur set: s = 16^3 - 14^3 = 1352, a FETI-style
              subdomain whose interior is eliminated; B = 16 and 64;
  p12_faces   Poisson 12^3 with its boundary, s = 728; B = 256;
  fem18_top   FEM 18^3 nodes x 3 dof (27-point), the top separator of the geometric nested dissection (s = 972; the case
              tests/test_schur_symbolic_cpu._fem18_w512, maxsup 512 in double, 256 in doublecomplex); B = 8.
The Schur set is numbered last by hostlib.schur_order (a nested dissection of the rest); relax 64, maxsup 256 (512 for
fem18_top in double).  Values: the non-symmetric, diagonally dominant matrix of scripts/bench_solve_trans.py, one member
per matgen.batch_values seed.  Per timed round and member set: fill_csr + factor, schur_get, condense + expand in each arm:
  batched arm:     batch_fill_csr, batch_factor, batch_schur_get, batch_schur_condense, batch_schur_expand on ONE handle;
  sequential arm:  fill_csr, factor, schur_get, schur_condense, schur_expand member after member on one Schur handle.
Times: factor = stats.t_factor_s (device events), gather = stats.reserved[7] (device events around the gather kernel),
schur_get = stats.reserved[6] (host clock around the call: memset, gather, D2H into pageable memory; both arms write into
one B x s x s host buffer touched before the timed rounds, member j's S at block j), condense + expand =
stats.reserved[4] of each (host clock, H2D of b and D2H of x included); the sequential arm sums over the members; medians
over the timed rounds, reported whole and per member.  Checks, outside the timed rounds: every member's composed solve
(condense, x2 = S_j^-1 g_j by numpy, expand) has ||F_j x - b|| / (||F_j|| ||x|| + ||b||) <= 1e-12, and the batched S of
members 0 and B - 1 equals the sequential arm's to 1e-12.  Prints one JSON line per (workload, B) with the launch counts
of both arms and the card's name and power limit read in the same run.  One GPU; writes nothing to disk.
"""
import argparse
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
from bench_solve_trans import gpu_name_and_power, values  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib, matgen  # noqa: E402

WORKLOADS = {"p16_faces": [16, 64], "p12_faces": [256], "fem18_top": [8]}


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--batch", type=int, nargs="+", default=None, help="members (default: the workload's own list)")
    ap.add_argument("--dtype", default="f64", choices=["f64", "c128"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if a.batch and min(a.batch) < 1:
        ap.error("--batch must be >= 1")
    return a


def faces(g):
    """the boundary nodes of a g^3 grid (x fastest)"""
    i = np.arange(g ** 3)
    x, y, z = i % g, (i // g) % g, i // (g * g)
    return i[(x == 0) | (x == g - 1) | (y == 0) | (y == g - 1) | (z == 0) | (z == g - 1)]


def problem(name, cplx):
    """-> (rp, ci, v, LUProblem with layer 0, s, description of the Schur set)"""
    if name == "fem18_top":
        rp, ci, v = hostlib.fem3d(18, dof=3)
        nd = hostlib.nd_order(18, dof=3, leaf=32)
        schur = np.argsort(nd)[len(rp) - 1 - 972:]                    # the top separator, in the ND's order
        maxsup, what = (256 if cplx else 512), "top-level separator of the geometric ND (FEM 18^3 x 3 dof)"
    else:
        g = 16 if name == "p16_faces" else 12
        rp, ci, v = hostlib.poisson3d(g)
        schur = faces(g)
        maxsup, what = 256, f"the six boundary faces of Poisson {g}^3"
    s = len(schur)
    perm = hostlib.schur_order(rp, ci, schur, leaf=8)
    sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=64, maxsup=maxsup, amalg=0.05, nschur=s)
    prob = LUProblem.from_symbolic(sym, npdep=1)
    if cplx:
        prob.dtype = np.dtype(np.complex128)
    prob.add_layer(0)
    return rp, ci, v, prob, s, what, maxsup


def run_one(name, nb, args, gpu):
    import scipy.sparse as sp
    cplx = args.dtype == "c128"
    rp, ci, v, prob, s, what, maxsup = problem(name, cplx)
    n, n1 = prob.n, prob.n - s
    vals = matgen.batch_values(rp, ci, values(rp, ci, v, cplx), nb, seed=0)
    pm = np.asarray(prob.perm, np.int32)
    b = np.random.default_rng(4).standard_normal((nb, n))
    if cplx:
        b = b + 1j * np.random.default_rng(5).standard_normal((nb, n))
    med = lambda xs: float(np.median(xs))  # noqa: E731
    # both arms write S into this one host buffer, touched before the timed rounds (fresh pageable memory would add its
    # page faults to every copy)
    host = np.empty((nb, s, s), prob.dtype)
    host.fill(0)

    # batched arm
    bh = capi.BatchSchurHandle(prob, nb, s, device=0)
    tb = {k: [] for k in ("factor", "gather", "schur_get", "condense_expand")}
    for i in range(args.warmup + args.steps):
        bh.fill_csr(rp, ci, vals, pm)
        assert not bh.factor().any()
        tf = bh.stats().t_factor_s
        S = bh.schur(out=host)
        st = bh.stats()
        y = bh.condense(b)
        tc = bh.stats().reserved[4]
        x = bh.expand(y)
        if i >= args.warmup:
            tb["factor"].append(tf)
            tb["gather"].append(st.reserved[7] * 1e-3)
            tb["schur_get"].append(st.reserved[6])
            tb["condense_expand"].append(tc + bh.stats().reserved[4])
    sb = bh.stats()
    launches_b = {"factor": int(sb.gpu_launches), "expand": int(sb.reserved[5])}
    # the composed solve of every member, outside the timed rounds
    y = bh.condense(b)
    launches_b["condense"] = int(bh.stats().reserved[5])
    y[:, n1:] = np.linalg.solve(S, y[:, n1:, None])[..., 0]
    x = bh.expand(y)
    rows = np.repeat(np.arange(n), np.diff(rp))
    res = 0.0
    for j in range(nb):
        F = sp.csr_matrix((vals[j], (pm[rows], pm[ci])), shape=(n, n))
        r = np.linalg.norm(F @ x[j] - b[j]) / (abs(F).sum(axis=1).max() * np.linalg.norm(x[j]) + np.linalg.norm(b[j]))
        res = max(res, float(r))
    assert res <= 1e-12, f"composed solve residual {res}"
    S_check = {j: S[j].copy() for j in sorted({0, nb - 1})}
    del S
    bh.close()

    # sequential arm: one unbatched Schur handle, member after member
    h = capi.SchurHandle(prob, s, device=0)
    get = getattr(capi.lib(), ("slu_b200_z_" if cplx else "slu_b200_") + "schur_get")
    ts = {k: [] for k in tb}
    for i in range(args.warmup + args.steps):
        acc = dict.fromkeys(tb, 0.0)
        for j in range(nb):
            h.fill_csr(rp, ci, vals[j], pm)
            assert h.factor() == 0
            acc["factor"] += h.stats().t_factor_s
            assert get(h.h, host[j].ctypes.data_as(ctypes.c_void_p), s) == 0    # S_j^T in host[j]
            Sj = host[j].T
            st = h.stats()
            acc["gather"] += st.reserved[7] * 1e-3
            acc["schur_get"] += st.reserved[6]
            yj = h.condense(b[j])
            tc = h.stats().reserved[4]
            h.expand(yj)
            acc["condense_expand"] += tc + h.stats().reserved[4]
            if j in S_check and i == args.warmup + args.steps - 1:
                err = np.abs(Sj - S_check[j]).max() / np.abs(S_check[j]).max()
                assert err <= 1e-12, f"member {j}: batched against sequential S {err}"
        if i >= args.warmup:
            for k in tb:
                ts[k].append(acc[k])
    s1 = h.stats()
    launches_s = {"factor": int(s1.gpu_launches), "expand": int(s1.reserved[5])}
    h.condense(b[0])
    launches_s["condense"] = int(h.stats().reserved[5])
    nlevels = int(s1.nlevels)
    h.close()

    def arm(k):
        bm, sm = med(tb[k]), med(ts[k])
        return {"batched_ms": round(bm * 1e3, 4), "sequential_ms": round(sm * 1e3, 4),
                "batched_ms_per_member": round(bm / nb * 1e3, 4), "sequential_ms_per_member": round(sm / nb * 1e3, 4),
                "speedup_per_member": round(sm / bm, 3)}

    print(bench.json_line({
        "metric": "batched_schur_factor_ms_per_member", "value": arm("factor")["batched_ms_per_member"], "unit": "ms",
        "higher_is_better": False, "workload": name, "schur_set": what, "n": n, "s": s, "batch": nb, "dtype": args.dtype,
        "maxsup": maxsup, "nlevels": nlevels, "steps": args.steps, "warmup": args.warmup,
        "values": "non-symmetric, diagonally dominant (scripts/bench_solve_trans.py), matgen.batch_values per member",
        "factor": arm("factor"), "gather": arm("gather"), "schur_get": arm("schur_get"),
        "condense_expand": arm("condense_expand"), "ops_fact_per_member": s1.ops_fact,
        "gpu_launches": {"batched": launches_b, "unbatched": launches_s},
        "composed_solve_max_residual": res, "gpu": gpu,
        "how": "factor: stats.t_factor_s; gather: stats.reserved[7] (device events); schur_get: stats.reserved[6] (host "
               "clock, D2H included); condense + expand: stats.reserved[4] (host clock, transfers included); sequential = "
               "sum over the members; medians of the timed rounds"}))


def main():
    args = parse()
    capi.require_gpu()
    gpu = gpu_name_and_power()
    for name in args.workloads:
        for nb in args.batch or WORKLOADS[name]:
            run_one(name, nb, args, gpu)


if __name__ == "__main__":
    main()
