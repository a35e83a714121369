"""Iterative refinement on the caller's stream (slu_b200_gsrfs_device, its loop in conditional graph nodes) against the host
loop of slu_b200_gsrfs, which reads a counter back after every step and every estimator round.

    python scripts/bench_refine_device.py [--reps R] [--only NAME]

Workloads: bench_refine.py's fem3 40^3 x 3 and KKT [K B^T; B 0] (2D Poisson K on 200^2, 10 000 constraints), where the
solves dominate, and Poisson 16^3 with B = 256 members, where the per-step waits of the host loop are the largest share.
One right-hand side per member, refined from solve_scaled's x with the forward error bound (ferr).  Arms per iteration:
  * host: gsrfs on host b and x (their H2D and D2H copies included);
  * device: gsrfs_device on CUDA tensors, eager (the handle's cached graph), then a device synchronise;
  * graph: one torch.cuda.CUDAGraph of refill -> factor_device -> solve_scaled_device -> gsrfs_device on the same values,
    captured once after a warm-up and replayed (this arm also refactors and solves).
One JSON line per workload, with the GPU's name and power limit read in the same run: the median iteration time of each arm
(host clock around work that ends in a device synchronise; the arms alternate, R iterations per arm and round, two rounds),
the refinement steps, the launches of gsrfs_device, and the largest relative difference of the device arms' x from the host
arm's.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_device_io import gpu_info, median_time, workload  # noqa: E402
from bench_refine import handle  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402
from test_static_pivot_cpu import csr_parts, kkt  # noqa: E402

WORKLOADS = ["fem3", "kkt", "poisson16"]


def build(name):
    """(tag, handle, rp, ci, values as the handle's scaled fill took them, batch or None)"""
    if name == "fem3":
        g = 40
        rp, ci, v = hostlib.fem3d(g, g, g, dof=3)
        n = len(rp) - 1
        h, _ = handle(rp, ci, v, lambda pr, prp, pci: hostlib.nd_order(g, dof=3, leaf=8) if np.array_equal(pr, np.arange(n))
                      else hostlib.nd_order_graph(prp, pci, leaf=64))
        return f"fem3-{g}^3x3", h, rp, ci, v, None
    if name == "kkt":
        rp, ci, v = csr_parts(kkt(200, 10000, 1))
        h, _ = handle(rp, ci, v, lambda pr, prp, pci: hostlib.nd_order_graph(prp, pci, leaf=64))
        return "kkt-poisson200^2-10000", h, rp, ci, v, None
    tag, rp, ci, v, perm, B = workload(name)
    n = len(rp) - 1
    prob = LUProblem.from_matrix(rp, ci, v, perm, relax=32, maxsup=256)
    h = capi.BatchHandle(prob, B)
    vals = np.stack([v] * B)
    h.fill_csr_scaled(rp, ci, vals, prob.perm, np.arange(n, dtype=np.int32), equil=True)
    assert (h.factor() == 0).all()
    return f"{tag}-B{B}", h, rp, ci, vals, B


def run(name, reps, info):
    tag, h, rp, ci, vals, B = build(name)
    n = len(rp) - 1
    batched = B is not None
    rng = np.random.default_rng(0)
    b = rng.standard_normal((B, n) if batched else (n,))
    x0 = h.solve_scaled(b)
    dev = torch.device("cuda")
    bd, x0d = torch.from_numpy(b).to(dev), torch.from_numpy(x0).to(dev)
    sv = torch.from_numpy(np.ascontiguousarray(vals)).to(dev)
    info_t = torch.zeros((B,) if batched else (1,), dtype=torch.int32, device=dev)

    def host_arm():
        return h.refine(b, x0)

    def device_arm():
        out = h.refine(bd, x0d)
        torch.cuda.synchronize()
        return out

    def iteration():
        h.refill(sv)
        h.factor_device(info_t)
        return h.refine(bd, h.solve_scaled(bd))

    xh, berr_h, steps_h, _ = host_arm()
    xd, berr_d, steps_d, _ = device_arm()
    launches = int(h.stats().reserved[5])
    side = torch.cuda.Stream()              # warm-up of the captured calls on a side stream, as torch recommends
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        iteration()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = iteration()

    def graph_arm():
        g.replay()
        torch.cuda.synchronize()
        return out

    xg, _, steps_g, _ = graph_arm()
    assert (info_t.cpu().numpy() == 0).all()
    scale = np.abs(xh).max()
    d_dev = float(np.abs(xd.cpu().numpy() - xh).max() / scale)
    d_graph = float(np.abs(xg.cpu().numpy() - xh).max() / scale)
    t = {"host": 0.0, "device": 0.0, "graph": 0.0}
    for _ in range(2):      # alternate the arms
        for k, fn in (("host", host_arm), ("device", device_arm), ("graph", graph_arm)):
            t[k] += median_time(fn, reps) / 2
    print(json.dumps({"workload": tag, "n": n, "nnz": len(ci), "batch": B or 1,
                      "iter_host_ms": t["host"] * 1e3, "iter_device_ms": t["device"] * 1e3, "iter_graph_ms": t["graph"] * 1e3,
                      "steps_host_max": int(np.max(steps_h)), "steps_device_max": int(steps_d.max()),
                      "steps_graph_max": int(steps_g.max()), "berr_max": float(berr_d.max()), "launches_device": launches,
                      "x_rel_diff_device": d_dev, "x_rel_diff_graph": d_graph, **info}), flush=True)
    del g
    h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", choices=WORKLOADS)
    a = ap.parse_args()
    info = gpu_info()
    for name in ([a.only] if a.only else WORKLOADS):
        run(name, a.reps, info)


if __name__ == "__main__":
    main()
