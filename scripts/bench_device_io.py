"""Refactorization with values and right-hand sides that live on the GPU: the device-resident calls (slu_b200_refill,
_solve_scaled_device and their batched twins) against the host calls they replace.

    python scripts/bench_device_io.py [--reps R] [--only NAME]

Per iteration both arms get new values (every entry times 1 + 0.01 u) and a new b, generated on the device with torch:
  * device arm: refill -> factor -> solve_scaled on the CUDA tensors (slu_b200_[batch_]refill, _solve_scaled_device);
  * host arm: values and b copied to the host -> fill_csr_scaled with the kept R and C and no EQUIL -> factor ->
    solve_scaled -> x copied back to the device.
Workloads: fem3 40^3 x 3 (n = 192 000, nnz 14.8 M; the matrix of bench_scaled.py and bench_refine.py), Poisson 32^3 with
B = 64, Poisson 16^3 with B = 256.  One JSON line per workload, with the GPU's name and power limit read in the same run:
  * the median iteration time of each arm (host clock around the iteration, which ends in a device synchronise);
  * the median fill call alone of each arm (refill + synchronise; the D2H of the values + fill_csr_scaled);
  * the device time of refill_kernel and fill_scaled_kernel on the same values, from torch.profiler's CUDA activities in a
    separate phase after the timed loops (the scaled fill's kernel cannot be bracketed by events from outside the call);
  * the bytes each arm moves over PCIe per iteration, computed from the sizes;
  * the largest relative difference between the two arms' x on the same values.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["unknown, unknown"])[0].split(", ")
    return {"gpu": name, "power_limit": power}


def median_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def workload(name):
    """(tag, rowptr, colind, values, perm, batch or None)"""
    if name == "fem3":
        rp, ci, v = hostlib.fem3d(40, 40, 40, dof=3)
        return "fem3-40^3x3", rp, ci, v, hostlib.nd_order(40, dof=3, leaf=8), None
    g, B = {"poisson32": (32, 64), "poisson16": (16, 256)}[name]
    rp, ci, v = hostlib.poisson3d(g)
    return f"poisson{g}^3", rp, ci, v, hostlib.nd_order(g, leaf=8), B


def kernel_ms(prof, key):
    """mean device ms of the kernels whose name contains key"""
    ts = [e.device_time_total / max(e.count, 1) for e in prof.key_averages() if key in e.key and e.count]
    return ts[0] * 1e-3 if ts else float("nan")


def run(name, reps, info):
    tag, rp, ci, v, perm, B = workload(name)
    n, nnz = len(rp) - 1, len(ci)
    prob = LUProblem.from_matrix(rp, ci, v, perm, relax=32, maxsup=256)
    perm_r = np.arange(n, dtype=np.int32)
    batched = B is not None
    mem = B or 1
    h = capi.BatchHandle(prob, B) if batched else capi.Handle(prob, 0)
    base = np.stack([v] * B) if batched else v
    h.fill_csr_scaled(rp, ci, base, prob.perm, perm_r, equil=True)
    if batched:
        RC = [h.scaling(j) for j in range(B)]
        R, C = np.stack([r for r, _ in RC]), np.stack([c for _, c in RC])
    else:
        _, R, C = h.scaling()
    dev = torch.device("cuda")
    vbase = torch.from_numpy(np.ascontiguousarray(base)).to(dev)
    bshape = (B, n) if batched else (n,)
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)

    def new_values():
        return vbase * (1.0 + 0.01 * torch.rand(vbase.shape, generator=gen, device=dev, dtype=torch.float64))

    def new_b():
        return torch.rand(bshape, generator=gen, device=dev, dtype=torch.float64)

    def factor():
        info_ = h.factor()
        assert (np.asarray(info_) == 0).all()

    def device_iter(vals=None, b=None):
        h.refill(new_values() if vals is None else vals)
        factor()
        return h.solve_scaled(new_b() if b is None else b)

    def host_iter(vals=None, b=None):
        vh = (new_values() if vals is None else vals).cpu().numpy()
        bh = (new_b() if b is None else b).cpu().numpy()
        h.fill_csr_scaled(rp, ci, vh, prob.perm, perm_r, R, C, equil=False)
        factor()
        return torch.from_numpy(h.solve_scaled(bh)).to(dev)

    # the same values and b through both arms
    vals, b = new_values(), new_b()
    xd = device_iter(vals, b).cpu().numpy()
    xh = host_iter(vals, b).cpu().numpy()
    diff = float(np.abs(xd - xh).max() / np.abs(xh).max())

    t_dev = t_host = 0.0
    for _ in range(2):      # alternate the arms
        t_dev += median_time(device_iter, reps) / 2
        t_host += median_time(host_iter, reps) / 2
    vals = new_values()
    t_refill = median_time(lambda: h.refill(vals), reps)
    launches = int(h.stats().reserved[5])
    t_fill = median_time(lambda: h.fill_csr_scaled(rp, ci, vals.cpu().numpy(), prob.perm, perm_r, R, C, equil=False), reps)
    vh = vals.cpu().numpy()
    t_fill_call = median_time(lambda: h.fill_csr_scaled(rp, ci, vh, prob.perm, perm_r, R, C, equil=False), reps)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            h.refill(vals)
            h.fill_csr_scaled(rp, ci, vh, prob.perm, perm_r, R, C, equil=False)
        torch.cuda.synchronize()
    k_refill, k_fill = kernel_ms(prof, "refill_kernel"), kernel_ms(prof, "fill_scaled_kernel")

    vbytes, bbytes = 8 * nnz * mem, 8 * n * mem
    # host arm: values and b down; rowptr, colind, values, perm_r / rmap / perm, R and C up (fill_csr_scaled); b up and x down
    # (solve_scaled); x up
    host_pcie = vbytes + bbytes + (4 * (n + 1) + 4 * nnz + vbytes + 12 * n + 2 * 8 * n * mem) + 2 * bbytes + bbytes
    print(json.dumps({"workload": tag, "n": n, "nnz": nnz, "batch": mem, "iter_device_ms": t_dev * 1e3, "iter_host_ms": t_host * 1e3,
                      "fill_device_ms": t_refill * 1e3, "fill_host_ms": t_fill * 1e3, "fill_host_call_only_ms": t_fill_call * 1e3,
                      "refill_kernel_ms": k_refill, "fill_scaled_kernel_ms": k_fill, "refill_launches": launches,
                      "pcie_bytes_device": 0, "pcie_bytes_host": host_pcie, "x_rel_diff": diff, **info}), flush=True)
    h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", choices=["fem3", "poisson32", "poisson16"])
    a = ap.parse_args()
    info = gpu_info()
    for name in ([a.only] if a.only else ["fem3", "poisson32", "poisson16"]):
        run(name, a.reps, info)


if __name__ == "__main__":
    main()
