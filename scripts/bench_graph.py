"""Refill -> factor -> solve with the factorization on the caller's stream, and the whole iteration as one CUDA graph:
slu_b200_factor_device (and its batched twin) against slu_b200_factor, which waits for the GPU.

    python scripts/bench_graph.py [--reps R] [--only NAME]

Per iteration every arm copies new values (every entry times 1 + 0.01 u) and a new b, generated on the device with torch,
into the same two tensors, then:
  * host_wait: refill -> factor (host wait, info read on the host) -> solve_scaled on the tensors;
  * device: refill -> factor_device -> solve_scaled, no host wait inside the iteration;
  * graph: one torch.cuda.CUDAGraph of the device arm, captured once after a warm-up and replayed.
Workloads: those of bench_device_io.py (fem3 40^3 x 3, Poisson 32^3 with B = 64, Poisson 16^3 with B = 256) and Poisson
16^3 unbatched, where the host's launch work is the largest share.  One JSON line per workload, with the GPU's name and
power limit read in the same run: the median iteration time of each arm (host clock around the iteration, which ends in
a device synchronise; the arms alternate), the kernel launches per iteration, and the largest relative difference of each
arm's x from the host_wait arm's on the same values.
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

from bench_device_io import gpu_info, median_time, workload  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402

WORKLOADS = ["fem3", "poisson32", "poisson16", "poisson16u"]


def run(name, reps, info):
    if name == "poisson16u":
        rp, ci, v = hostlib.poisson3d(16)
        tag, perm, B = "poisson16^3", hostlib.nd_order(16, leaf=8), None
    else:
        tag, rp, ci, v, perm, B = workload(name)
    n, nnz = len(rp) - 1, len(ci)
    prob = LUProblem.from_matrix(rp, ci, v, perm, relax=32, maxsup=256)
    perm_r = np.arange(n, dtype=np.int32)
    batched = B is not None
    h = capi.BatchHandle(prob, B) if batched else capi.Handle(prob, 0)
    base = np.stack([v] * B) if batched else v
    h.fill_csr_scaled(rp, ci, base, prob.perm, perm_r, equil=True)
    dev = torch.device("cuda")
    vbase = torch.from_numpy(np.ascontiguousarray(base)).to(dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    sv = vbase.clone()
    sb = torch.zeros((B, n) if batched else (n,), dtype=torch.float64, device=dev)
    info_t = torch.zeros((B,) if batched else (1,), dtype=torch.int32, device=dev)

    def new_inputs():
        sv.copy_(vbase * (1.0 + 0.01 * torch.rand(vbase.shape, generator=gen, device=dev, dtype=torch.float64)))
        sb.copy_(torch.rand(sb.shape, generator=gen, device=dev, dtype=torch.float64))

    def host_wait(inputs=True):
        if inputs:
            new_inputs()
        h.refill(sv)
        assert (np.asarray(h.factor()) == 0).all()
        return h.solve_scaled(sb)

    def device(inputs=True):
        if inputs:
            new_inputs()
        h.refill(sv)
        h.factor_device(info_t)
        return h.solve_scaled(sb)

    h.refill(sv)                        # the slot map, once per scaled fill: not part of an iteration
    # launches per iteration: refill + factorization + solve, from the stats of each call
    def launches(fact):
        h.refill(sv)
        n_refill = int(h.stats().reserved[5])
        fact()
        n_fact = int(h.stats().gpu_launches)
        h.solve_scaled(sb)
        return n_refill + n_fact + int(h.stats().reserved[5])
    l_host = launches(h.factor)
    l_dev = launches(lambda: h.factor_device(info_t))

    side = torch.cuda.Stream()          # warm-up of the captured calls on a side stream, as torch recommends
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        device(False)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sx = device(False)

    def graph(inputs=True):
        if inputs:
            new_inputs()
        g.replay()
        return sx

    # the same values and b through the three arms
    new_inputs()
    x_host = host_wait(False).cpu().numpy()
    x_dev = device(False).cpu().numpy()
    x_graph = graph(False).cpu().numpy()
    torch.cuda.synchronize()
    assert (info_t.cpu().numpy() == 0).all()
    scale = np.abs(x_host).max()
    d_dev, d_graph = float(np.abs(x_dev - x_host).max() / scale), float(np.abs(x_graph - x_host).max() / scale)

    t = {"host_wait": 0.0, "device": 0.0, "graph": 0.0}
    for _ in range(2):      # alternate the arms
        for k, fn in (("host_wait", host_wait), ("device", device), ("graph", graph)):
            t[k] += median_time(fn, reps) / 2
    print(json.dumps({"workload": tag, "n": n, "nnz": nnz, "batch": B or 1,
                      "iter_host_wait_ms": t["host_wait"] * 1e3, "iter_device_ms": t["device"] * 1e3, "iter_graph_ms": t["graph"] * 1e3,
                      "launches_host_wait": l_host, "launches_device": l_dev, "launches_graph": l_dev,
                      "x_rel_diff_device": d_dev, "x_rel_diff_graph": d_graph, "agree_1e-14": max(d_dev, d_graph) <= 1e-14, **info}),
          flush=True)
    del g
    h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--only", choices=WORKLOADS)
    a = ap.parse_args()
    info = gpu_info()
    for name in ([a.only] if a.only else WORKLOADS):
        run(name, a.reps, info)


if __name__ == "__main__":
    main()
