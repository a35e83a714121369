"""Deferred Schur updates along supernode chains (DESIGN 4a), CPU only: for a workload and deferral depths D, the count of
children whose update their parent's carries, the destination updates (RED.ADD.F64) of one factorization and the ratio
to D = 1 (slu_b200_k_schur_merge on the library's own analysis, slu_b200_plan's).  One JSON line per D.
    python scripts/schur_merge_plan.py [--workload fem3|poisson] [--grid G] [--maxsup 256] [--relax 64] [--leaf 64] [--depths 1,2,3,4]
Defaults: the bench.py workload (fem3, G = 68: n = 943,296)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superlu_dist_b200 import LUProblem, capi, hostlib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="fem3", choices=["fem3", "poisson"])
ap.add_argument("--grid", type=int, default=0)
ap.add_argument("--maxsup", type=int, default=256)
ap.add_argument("--relax", type=int, default=64)
ap.add_argument("--leaf", type=int, default=64)
ap.add_argument("--depths", default="1,2,3,4")
a = ap.parse_args()
g = a.grid or (68 if a.workload == "fem3" else 128)
t0 = time.time()
if a.workload == "fem3":   # as bench.py builds it
    rp, ci, v = hostlib.fem3d(g, g, g, dof=3)
    perm = hostlib.nd_order(g, dof=3, leaf=max(1, a.leaf // 3))
else:
    rp, ci, v = hostlib.poisson3d(g)
    perm = hostlib.nd_order(g, leaf=a.leaf)
sym = hostlib.Symbolic(len(rp) - 1, rp, ci, perm, a.relax, a.maxsup, 0.05)
prob = LUProblem.from_symbolic(sym)
del sym
prob.add_layer(0)   # untouched (lazily zero) arrays: only their addresses enter the view
t_sym = time.time() - t0
os.environ.pop("SLU_B200_SCHUR_DEPTH", None)
for d in (int(x) for x in a.depths.split(",")):
    deferred, reds1, reds = capi.schur_merge(prob, schur_depth=d)
    print(json.dumps({"workload": a.workload, "grid": g, "n": prob.n, "nsupers": prob.nsupers, "maxsup": a.maxsup, "depth": d,
                      "deferred_children": deferred, "reds": reds, "reds_depth1": reds1, "ratio": round(reds / reds1, 4),
                      "symbolic_s": round(t_sym, 1)}), flush=True)
