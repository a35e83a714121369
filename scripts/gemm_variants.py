"""Micro-benchmark of the DMMA main-loop tile configurations (slu_b200_k_gemm_sub, RED epilogue)."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, ".")
from superlu_dist_b200 import capi  # noqa: E402

NAMES = {0: "128x64 4x2w BK16 S3 (default)", 1: "128x64 BK16 S4", 2: "128x64 BK32 S2", 3: "128x128 4x4w BK16 S3 1CTA",
         4: "128x64 2x4w BK16 S3", 5: "64x64 2x2w BK16 S4", 6: "128x64 BK8 S4", 8: "128x128 2x4w (warp 64x32) 1CTA",
         9: "128x64 2x2w (warp 64x32) 2CTA", 10: "256x64 4x2w (warp 64x32)", 11: "128x128 4x2w (warp 32x64)",
         12: "128x128 4x4w S4", 13: "128x128 2x4w BK32 S2",
         # strength-reduced loader (gemm_tile_v2), opt-in
         14: "v2 128x64 BK16 S3", 15: "v2 128x64 BK32 S2", 16: "v2 128x64 BK16 S4", 17: "v2 32x32",
         18: "v2 128x128 4x2w (warp 32x64) 1CTA", 19: "v2 128x128 4x4w 1CTA",
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
