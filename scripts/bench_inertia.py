"""Spectrum slicing and affine fills on batched handles (slu_b200_batch_fill_affine, slu_b200_batch_inertia) against a
sequential loop of one unbatched handle.

    python scripts/bench_inertia.py [--configs poisson:16,poisson:32,fem3:12] [--batches 1,8,64] [--steps K] [--warmup W]

Per workload (Poisson 16^3 and 32^3, the 27-point fem3 at 12^3 nodes x 3 dof symmetrised as (A + A^T) / 2; nested
dissection, maxsup 256) and batch B, the eigenvalues of K below B shifts sigma_j spread over (0, ||K||_inf / 2) are counted:
  batched arm:     fill_affine(K, I; 1, -sigma_j), batch_factor, batch_inertia on ONE batched handle;
  sequential arm:  per shift the host builds K - sigma_j I, then fill_csr, factor, inertia on one unbatched handle.
Each arm's time is a host clock around its calls (every call ends in a stream synchronise); medians over the timed rounds,
whole and per member.  The counts of both arms must agree.  Fill cost: batch_fill_affine against batch_fill_csr of the
same B members on one batched handle, call time (host clock around the synchronised call) and the bytes each copies host
to device.  Prints one JSON line per (workload, B) with the card's name and power limit read in the same run.  One GPU;
writes nothing to disk.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_solve_trans import gpu_name_and_power  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="poisson:16,poisson:32,fem3:12", help="workload:grid, comma-separated")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    return ap.parse_args()


def workload(kind, g):
    """(rowptr, colind, symmetric values, nested-dissection perm)"""
    if kind == "fem3":
        rp, ci, v = hostlib.fem3d(g, g, g, dof=3)
        perm = hostlib.nd_order(g, dof=3, leaf=21)
        A = sp.csr_matrix((v, ci, rp), shape=(len(rp) - 1,) * 2)
        S = ((A + A.T) * 0.5).tocsr()
        S.sort_indices()
        if not (np.array_equal(S.indptr, rp) and np.array_equal(S.indices, ci)):
            raise RuntimeError("fem3d pattern is not structurally symmetric")
        return rp, ci, S.data.copy(), perm
    rp, ci, v = hostlib.poisson3d(g)
    return rp, ci, v, hostlib.nd_order(g, leaf=64)


def h2d_bytes(n, nnz, terms):
    """rowptr, colind, perm and the values (terms x nnz doubles) of one fill call"""
    return 4 * (n + 1) + 4 * nnz + 4 * n + 8 * terms * nnz


def run_config(kind, g, B, args, gpu):
    rp, ci, v, perm = workload(kind, g)
    n, nnz = len(rp) - 1, len(ci)
    rows = np.repeat(np.arange(n), np.diff(rp))
    eye = (rows == ci).astype(np.float64)
    bound = np.max(np.bincount(rows, np.abs(v), n))
    # off every round number: the leading blocks of these matrices have many (Poisson: integer) eigenvalues, where an
    # unpivoted factorization meets (near) zero pivots and two roundings may count differently
    sig = (np.arange(B) + 0.5 + 0.1 * np.sqrt(2.0)) / B * 0.5 * bound
    sym = hostlib.Symbolic(n, rp, ci, perm, relax=64, maxsup=256, amalg=0.05)
    prob = LUProblem.from_symbolic(sym, npdep=1)
    del sym
    prob.add_layer(0)
    pm = np.asarray(prob.perm, np.int32)
    terms, coef = np.stack([v, eye]), np.stack([np.ones(B), -sig], axis=1)
    med = lambda xs: float(np.median(xs))  # noqa: E731

    bh = capi.BatchHandle(prob, B, device=0)
    t_b, t_aff, t_csr = [], [], []
    members = np.ascontiguousarray(coef @ terms)
    for i in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        bh.fill_affine(rp, ci, terms, coef, pm)
        t1 = time.perf_counter()
        assert not bh.factor().any()
        neg_b = bh.inertia()[0]
        t2 = time.perf_counter()
        bh.fill_csr(rp, ci, members, pm)
        t3 = time.perf_counter()
        if i >= args.warmup:
            t_b.append(t2 - t0)
            t_aff.append(t1 - t0)
            t_csr.append(t3 - t2)
    bh.close()

    h = capi.Handle(prob, 0, device=0)
    t_s = []
    for i in range(args.warmup + args.steps):
        neg_s = np.zeros(B, np.int64)
        t0 = time.perf_counter()
        for j in range(B):
            h.fill_csr(rp, ci, v - sig[j] * eye, pm)
            assert h.factor() == 0
            neg_s[j] = h.inertia()[0]
        if i >= args.warmup:
            t_s.append(time.perf_counter() - t0)
    h.close()
    if not np.array_equal(neg_b, neg_s):
        raise RuntimeError(f"{kind} {g}^3 B={B}: counts differ between the arms: {neg_b} vs {neg_s}")
    return {"workload": f"{kind}-{g}^3" + ("-3dof-symmetrised" if kind == "fem3" else ""), "n": n, "nnz": nnz, "batch": B,
            "gpu": gpu, "counts": [int(x) for x in neg_b],
            "batched_s": med(t_b), "sequential_s": med(t_s), "batched_per_member_ms": 1e3 * med(t_b) / B,
            "sequential_per_member_ms": 1e3 * med(t_s) / B, "speedup": med(t_s) / med(t_b),
            "fill_affine_s": med(t_aff), "fill_csr_s": med(t_csr), "fill_speedup": med(t_csr) / med(t_aff),
            "fill_affine_h2d_bytes": h2d_bytes(n, nnz, 2) + 8 * 2 * B, "fill_csr_h2d_bytes": h2d_bytes(n, nnz, B)}


def main():
    args = parse()
    capi.require_gpu()
    gpu = gpu_name_and_power()
    for cfg in args.configs.split(","):
        kind, g = cfg.split(":")
        for B in (int(b) for b in args.batches.split(",")):
            print(json.dumps(run_config(kind, int(g), B, args, gpu)), flush=True)


if __name__ == "__main__":
    main()
