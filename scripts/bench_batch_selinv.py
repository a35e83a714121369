"""Selected inversion and log-determinants on a batched handle (slu_b200_batch_selinv, _batch_selinv_get, _batch_logdet)
against a sequential loop of one unbatched handle.

    python scripts/bench_batch_selinv.py --batch B [--dtype f64|c128] [--workload poisson|fem3] [--grid G]
                                         [--steps K] [--warmup W]

B matrices with the pattern of the bench.py workload at --grid (seeded values, matgen.batch_values; --dtype c128: the
members of scripts/bench_batch.py --dtype c128, the matrix with i * 0.5 * its diagonal added) are, per timed round,
filled on the device, factored, inverted on the pattern of L + U, and asked for the diagonal of A_j^-1 and log |det A_j|:
  batched arm:     batch_fill_csr, batch_factor, batch_selinv, inv_diag, logdet on ONE batched handle;
  sequential arm:  fill_csr, factor, selinv, inv_diag, logdet member after member on one unbatched handle.
Times: selinv = out[0] of the call (the library's host clock around the sweep; the sequential arm sums it over the members),
factor = stats.t_factor_s (device events), inv_diag and logdet = a host clock around the Python call (H2D of the pattern
and D2H of the values included); medians over the timed rounds, reported whole and per member.  Checks: inv_diag of
members 0 and B - 1 against 8 unit-vector batched solves (relative error <= 1e-10), and the batched log-determinants
against the sequential ones (relative <= 1e-12; signs equal, complex phases to 1e-12).  Prints one JSON line with the
launch counts of both arms and the card's name and power limit read in the same run.  One GPU; writes nothing to disk.
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
from bench_solve_trans import gpu_name_and_power  # noqa: E402
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
    a = ap.parse_args()
    if a.batch < 1:
        ap.error("--batch must be >= 1")
    return a


def run(args):
    capi.require_gpu()
    gpu = gpu_name_and_power()
    nb, G = args.batch, args.grid
    cplx = args.dtype == "c128"
    rp, ci, v, perm = bench.make_matrix(args, G)
    sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=args.relax, maxsup=args.maxsup, amalg=args.amalg)
    prob = LUProblem.from_symbolic(sym, npdep=1)
    del sym
    if cplx:
        prob.dtype = np.dtype(np.complex128)
        rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        v = v + 1j * np.where(rows == ci, 0.5 * v, 0.0)      # K + i w C with C = 0.5 diag(K), as bench_batch.py
    prob.add_layer(0)
    vals = matgen.batch_values(rp, ci, v, nb, seed=0)
    pm = np.asarray(prob.perm, np.int32)
    n = prob.n
    opt = dict(device=0)
    med = lambda xs: float(np.median(xs))  # noqa: E731

    # batched arm
    bh = capi.BatchHandle(prob, nb, **opt)
    tf_b, ts_b, td_b, tl_b = [], [], [], []
    for i in range(args.warmup + args.steps):
        bh.fill_csr(rp, ci, vals, pm)
        assert not bh.factor().any()
        tf = bh.stats().t_factor_s
        out_b = bh.selinv()
        t0 = time.perf_counter()
        d_b = bh.inv_diag(pm)
        t1 = time.perf_counter()
        sign_b, la_b = bh.logdet()
        t2 = time.perf_counter()
        if i >= args.warmup:
            tf_b.append(tf)
            ts_b.append(out_b[0])
            td_b.append(t1 - t0)
            tl_b.append(t2 - t1)
    launches_fb = int(bh.stats().gpu_launches)
    # inv_diag of members 0 and B - 1 against unit-vector solves (column perm[c] of F_j^-1 is column c of A_j^-1)
    cols = np.random.default_rng(2).choice(n, 8, replace=False)
    rhs = np.zeros((nb, 8, n), prob.dtype)
    rhs[:, np.arange(8), pm[cols]] = 1.0
    x = bh.solve(rhs)
    diag_err = 0.0
    for j in sorted({0, nb - 1}):
        ref = x[j, np.arange(8), pm[cols]]
        diag_err = max(diag_err, float(np.max(np.abs(d_b[j, cols] - ref) / np.abs(ref))))
    assert diag_err <= 1e-10, f"inv_diag against unit-vector solves: {diag_err}"
    hbm_b = int(out_b[3])
    bh.close()

    # sequential arm: one unbatched handle, member after member
    h = capi.Handle(prob, 0, tc_slices=-1, **opt)
    tf_s, ts_s, td_s, tl_s = [], [], [], []
    sign_s = np.zeros(nb, np.complex128 if cplx else np.float64)
    la_s = np.zeros(nb)
    for i in range(args.warmup + args.steps):
        tf = tsi = tdi = tlo = 0.0
        for j in range(nb):
            h.fill_csr(rp, ci, vals[j], pm)
            assert h.factor() == 0
            tf += h.stats().t_factor_s
            out_s = h.selinv()
            tsi += out_s[0]
            t0 = time.perf_counter()
            h.inv_diag(pm)
            t1 = time.perf_counter()
            sign_s[j], la_s[j] = h.logdet()
            tlo += time.perf_counter() - t1
            tdi += t1 - t0
        if i >= args.warmup:
            tf_s.append(tf)
            ts_s.append(tsi)
            td_s.append(tdi)
            tl_s.append(tlo)
    launches_fs, nlevels = int(h.stats().gpu_launches), int(h.stats().nlevels)
    h.close()
    logdet_err = float(np.max(np.abs(la_b - la_s) / np.abs(la_s)))
    sign_err = float(np.max(np.abs(sign_b - sign_s)))
    assert logdet_err <= 1e-12, f"batched against sequential log |det|: {logdet_err}"
    assert (sign_err <= 1e-12) if cplx else sign_err == 0.0, f"batched against sequential sign: {sign_err}"
    assert int(out_b[2]) == int(out_s[2]), (out_b[2], out_s[2])

    def arm(b, s):
        return {"batched_ms": round(med(b) * 1e3, 4), "sequential_ms": round(med(s) * 1e3, 4),
                "batched_ms_per_member": round(med(b) / nb * 1e3, 4), "sequential_ms_per_member": round(med(s) / nb * 1e3, 4),
                "speedup_per_member": round(med(s) / med(b), 3)}

    workload = bench.workload_name(G, args.workload, args.ordering)
    sel = arm(ts_b, ts_s)
    sel["gflops_batched"] = round(out_b[1] / med(ts_b) * 1e-9, 2)
    sel["gflops_sequential"] = round(nb * out_s[1] / med(ts_s) * 1e-9, 2)
    print(bench.json_line({
        "metric": "batched_selinv_ms_per_member", "value": sel["batched_ms_per_member"], "unit": "ms", "higher_is_better": False,
        "batch": nb, "steps": args.steps, "warmup": args.warmup, "dtype": args.dtype, "data": "synthetic",
        "workload": workload.replace("fp64", "c128") if cplx else workload, "n": n, "nlevels": nlevels,
        "selinv": sel, "factor": arm(tf_b, tf_s), "inv_diag": arm(td_b, td_s), "logdet": arm(tl_b, tl_s),
        "selinv_flops_per_member": out_s[1], "selinv_hbm_bytes_batched": hbm_b,
        "gpu_launches": {"batched_selinv": int(out_b[2]), "unbatched_selinv": int(out_s[2]),
                         "batched_factor": launches_fb, "unbatched_factor": launches_fs},
        "inv_diag_vs_solves_max_rel_err": diag_err, "logdet_batched_vs_sequential_max_rel_err": logdet_err,
        "sign_batched_vs_sequential_max_err": sign_err, "gpu": gpu,
        "how": "selinv: out[0] (host clock around the sweep; sequential = sum over the members); factor: stats.t_factor_s; "
               "inv_diag / logdet: host clock around the Python call; median of the timed rounds"}))


if __name__ == "__main__":
    run(parse())
