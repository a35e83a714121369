"""Gradients through the resident factors (superlu_dist_b200.autograd): the forward step and the two halves of its backward,
and the two gradient kernels against their byte bounds.

    python scripts/bench_autograd.py [--reps R] [--only NAME]

Per workload (values: the matrix's own, every entry times 1 + 0.01 u per iteration, generated on the device):
  * forward: autograd.factorize (refill + factor_device) -> Factors.solve -> Factors.slogdet;
  * backward_solve: the transposed solve_scaled of dL/dx and solve_grad (the SDDMM -lambda x^T on A's pattern);
  * backward_logdet: selinv_device and logdet_grad (the gather of coef * A^-T on A's pattern).  Selected inversion costs
    several factorizations (README), so it dominates this half;
  * kernel times of solve_grad_kernel and logdet_grad_kernel, from a torch.profiler phase of its own, against the time
    their algorithmic bytes take at 3.35 TB/s (the H100 SXM's HBM3 data-sheet bandwidth);
  * solve_grad against the torch expression -(lam[..., rows, :] * x[..., cols, :]).sum(-1) on the same lambda and x: time
    and the peak memory each allocates.
Host clock around synchronised work, medians after a warm-up, the arms alternating.  One JSON line per workload with the
GPU's name and power limit read in the same run.
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

from bench_device_io import gpu_info, kernel_ms, median_time  # noqa: E402
from superlu_dist_b200 import LUProblem, autograd, capi, hostlib  # noqa: E402

HBM_BPS = 3.35e12
# (name, grid, dof, batch, nrhs, complex)
WORKLOADS = {
    "fem3-n1": ("fem3", 40, 3, None, 1, False),
    "fem3-n8": ("fem3", 40, 3, None, 8, False),
    "poisson32-n1": ("poisson", 32, 1, None, 1, False),
    "poisson32-n8": ("poisson", 32, 1, None, 8, False),
    "poisson16-B64-n1": ("poisson", 16, 1, 64, 1, False),
    "poisson16-B64-n8": ("poisson", 16, 1, 64, 8, False),
    "poisson32-z-n8": ("poisson", 32, 1, None, 8, True),
}


def problem(kind, g, dof):
    if kind == "fem3":
        rp, ci, v = hostlib.fem3d(g, g, g, dof=dof)
        return f"fem3-{g}^3x{dof}", rp, ci, v, hostlib.nd_order(g, dof=dof, leaf=8)
    rp, ci, v = hostlib.poisson3d(g)
    return f"poisson{g}^3", rp, ci, v, hostlib.nd_order(g, leaf=8)


def run(key, reps, info):
    kind, g, dof, B, nrhs, cplx = WORKLOADS[key]
    tag, rp, ci, v, perm = problem(kind, g, dof)
    n, nnz = len(rp) - 1, len(ci)
    prob = LUProblem.from_matrix(rp, ci, v, perm, relax=32, maxsup=256)
    vals = v.astype(np.complex128) * (1 + 0.05j) if cplx else v
    if cplx:
        prob.dtype = np.dtype(np.complex128)
        for lay in prob.layers.values():
            lay.lval, lay.uval = lay.lval.astype(np.complex128), lay.uval.astype(np.complex128)
    h = capi.BatchHandle(prob, B) if B else capi.Handle(prob, 0)
    base = np.stack([vals] * B) if B else vals
    h.fill_csr_scaled(rp, ci, base, prob.perm, equil=True)
    dev = torch.device("cuda")
    dt = torch.complex128 if cplx else torch.float64
    vbase = torch.from_numpy(np.ascontiguousarray(base)).to(dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    lead = (B,) if B else ()
    bshape = lead + ((n,) if nrhs == 1 else (nrhs, n))
    sv = vbase.clone()
    sb = torch.rand(bshape, generator=gen, device=dev, dtype=torch.float64).to(dt)
    gx = torch.rand(bshape, generator=gen, device=dev, dtype=torch.float64).to(dt)
    coef = torch.ones(B or 1, dtype=dt, device=dev)
    state = {}

    def forward():
        sv.copy_(vbase * (1.0 + 0.01 * torch.rand(vbase.shape, generator=gen, device=dev, dtype=torch.float64)))
        f = autograd.factorize(h, sv)
        state["x"] = f.solve(sb)
        state["sl"] = f.slogdet()

    def backward_solve():
        lam = h.solve_scaled(gx, "H" if cplx else "T")
        state["lam"] = lam
        return h.solve_grad(lam, state["x"])

    def backward_logdet():
        h.selinv_device()
        return h.logdet_grad(coef)

    forward()
    backward_solve()
    backward_logdet()
    t = {"forward": 0.0, "backward_solve": 0.0, "backward_logdet": 0.0}
    for _ in range(2):
        t["forward"] += median_time(forward, reps) / 2
        t["backward_solve"] += median_time(backward_solve, reps) / 2
        t["backward_logdet"] += median_time(backward_logdet, reps) / 2
    forward()
    backward_solve()
    lam, x = state["lam"], state["x"]

    # the torch gather expression on the same lambda and x: (..., n, nrhs) rows
    rows = torch.from_numpy(np.repeat(np.arange(n), np.diff(rp))).to(dev)
    cols = torch.from_numpy(ci.astype(np.int64)).to(dev)
    L2 = (lam if nrhs > 1 else lam.unsqueeze(-2)).transpose(-1, -2)
    X2 = (x if nrhs > 1 else x.unsqueeze(-2)).transpose(-1, -2).conj()

    def torch_gather():
        return -(L2[..., rows, :] * X2[..., cols, :]).sum(-1)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        m0 = torch.cuda.memory_allocated()
        out = fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - m0, out

    mem_k, gk = peak(lambda: h.solve_grad(lam, x))
    mem_t, gt = peak(torch_gather)
    diff = float((gk.reshape(gt.shape) - gt).abs().max() / gt.abs().max())
    del gt
    tk = tt = 0.0
    for _ in range(2):
        tk += median_time(lambda: h.solve_grad(lam, x), reps) / 2
        tt += median_time(torch_gather, reps) / 2

    h.selinv_device()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            h.solve_grad(lam, x)
            h.logdet_grad(coef)
        torch.cuda.synchronize()
    members = B or 1
    vb = 16 if cplx else 8
    solve_bytes = members * (4 * nnz + 4 * (n + 1) + vb * nnz + 2 * vb * n * nrhs)
    logdet_bytes = members * (8 * nnz + 4 * nnz + 4 * nnz + vb * nnz + 2 * 8 * n + vb * nnz)
    ks, kl = kernel_ms(prof, "solve_grad_kernel"), kernel_ms(prof, "logdet_grad_kernel")
    print(json.dumps({"workload": tag, "n": n, "nnz": nnz, "batch": members, "nrhs": nrhs, "dtype": "complex128" if cplx else "float64",
                      "forward_ms": t["forward"] * 1e3, "backward_solve_ms": t["backward_solve"] * 1e3,
                      "backward_logdet_ms": t["backward_logdet"] * 1e3,
                      "solve_grad_kernel_ms": ks, "solve_grad_bound_ms": solve_bytes / HBM_BPS * 1e3,
                      "logdet_grad_kernel_ms": kl, "logdet_grad_bound_ms": logdet_bytes / HBM_BPS * 1e3,
                      "solve_grad_call_ms": tk * 1e3, "torch_gather_ms": tt * 1e3,
                      "solve_grad_peak_mb": mem_k / 2**20, "torch_gather_peak_mb": mem_t / 2**20, "solve_grad_vs_torch_rel": diff,
                      **info}), flush=True)
    h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", choices=list(WORKLOADS))
    a = ap.parse_args()
    capi.require_gpu()
    info = gpu_info()
    for key in ([a.only] if a.only else WORKLOADS):
        run(key, a.reps, info)


if __name__ == "__main__":
    main()
