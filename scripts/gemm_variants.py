"""Micro-benchmark of the DMMA main-loop tile configurations (slu_b200_k_gemm_sub, RED epilogue)."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, ".")
from superlu_dist_b200 import capi  # noqa: E402

NAMES = {0: "default (m, n >= 96: variant 30)",
         # the Hopper main loop (gemm_tile_h: DMMA.16x8x8, warp tile 64x32); 30 is the Schur path's tile
         30: "h 128x64 2x2w BK16 S3 2CTA", 31: "h 128x64 2x2w BK32 S2 2CTA", 32: "h 128x128 2x4w BK16 S4 1CTA",
         33: "h 128x128 2x4w BK32 S3 1CTA", 34: "h 64x64 1x2w BK16 S3 3CTA"}
if len(sys.argv) > 1:
    NAMES = {int(v): NAMES[int(v)] for v in sys.argv[1].split(",")}
rng = np.random.default_rng(0)
for (m, n, k) in [(8192, 8192, 256), (8192, 8192, 64)]:
    a, b, c = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((m, n))
    ref = None
    for v in sorted(NAMES):
        os.environ["SLU_B200_GEMM_VARIANT"] = str(v)
        out, ms = capi.k_gemm_sub(a, b, c, reps=10)
        if ref is None:
            ref = c - a @ b
        err = float(np.abs(out - ref).max())
        print(json.dumps({"m": m, "n": n, "k": k, "variant": v, "name": NAMES[v], "ms": round(ms, 4),
                          "tflops": round(2.0 * m * n * k / ms * 1e-9, 2), "max_err": err}), flush=True)
