"""Per-level timing of the FP64 Schur kernel on the bench workload: factor once, then re-run the Schur launches of the
N levels with the most big-tile flops (slu_b200_k_rerun_schur) and time the plain GEMM with the same main loop
(slu_b200_k_gemm_sub variant 30, RED epilogue into a dense C) at each level's flop-weighted (m, n, k).
    python scripts/schur_levels.py [--grid 68] [--workload fem3] [--levels 4] [--reps 3]
Prints the card, then one JSON line per level: level, supernodes, tiles, gflop, ms, tflops, gemm_sub_tflops."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--grid", type=int, default=68)
ap.add_argument("--workload", default="fem3", choices=["fem3", "poisson"])
ap.add_argument("--levels", type=int, default=4)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--leaf", type=int, default=64)
ap.add_argument("--maxsup", type=int, default=256)
ap.add_argument("--relax", type=int, default=64)
ap.add_argument("--ordering", default="geometric")
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(json.dumps({"card": card, "workload": bench.workload_name(args.grid, args.workload, args.ordering)}), flush=True)

rp, ci, v, perm = bench.make_matrix(args, args.grid)
sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, relax=args.relax, maxsup=args.maxsup, amalg=0.05)
prob = LUProblem.from_symbolic(sym, npdep=1)
prob.add_layer(0, alloc=capi.pinned_alloc)
prob.fill_layer(0, rp, ci, v)
# tc_slices = -1: every big update (m, n >= 96) on the FP64 kernel, so the level's flops are all this kernel's
h = capi.Handle(prob, 0, pinned=1, tc_slices=-1)
h.upload()
assert h.factor() == 0

ns = np.diff(np.asarray(prob.xsup)).astype(np.float64)
m = np.asarray(prob.lidx)[np.asarray(prob.lidx_off)[:-1] + 1].astype(np.float64) - ns
n = np.asarray(prob.uval_len, dtype=np.float64) / np.maximum(ns, 1)

L = capi.lib()
L.slu_b200_k_level_export.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
L.slu_b200_k_rerun_schur.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float)]
nodes = (C.c_int32 * (1 << 20))()
levels = []
for li in range(h.stats().nlevels):
    cnt = L.slu_b200_k_level_export(h.h, li, None, 0, nodes, len(nodes))
    if cnt <= 0:
        continue
    k = np.frombuffer(nodes, dtype=np.int32, count=cnt)
    fl = 2.0 * m[k] * n[k] * ns[k]
    tiles = int((np.ceil(m[k] / 128) * np.ceil(n[k] / 64)).sum())
    w = fl / fl.sum()
    levels.append((fl.sum(), li, cnt, tiles, [int(round((x[k] * w).sum())) for x in (m, n, ns)]))
levels.sort(reverse=True)

rng = np.random.default_rng(0)
for flops, li, cnt, tiles, (wm, wn, wk) in levels[:args.levels]:
    ms = C.c_float(0)
    if L.slu_b200_k_rerun_schur(h.h, li, args.reps, C.byref(ms)) != 0:
        raise SystemExit(L.slu_b200_last_error().decode())
    a, b, c = rng.standard_normal((wm, wk)), rng.standard_normal((wk, wn)), np.zeros((wm, wn))
    os.environ["SLU_B200_GEMM_VARIANT"] = "30"
    try:
        _, gms = capi.k_gemm_sub(a, b, c, reps=10)
    finally:
        os.environ.pop("SLU_B200_GEMM_VARIANT", None)
    print(json.dumps({"level": li, "supernodes": cnt, "tiles": tiles, "gflop": round(flops * 1e-9, 2),
                      "ms": round(ms.value, 3), "tflops": round(flops / ms.value * 1e-9, 2),
                      "gemm_sub_shape": [wm, wn, wk], "gemm_sub_tflops": round(2.0 * wm * wn * wk / gms * 1e-9, 2)}), flush=True)
h.close()
