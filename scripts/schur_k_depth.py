"""Time the Schur main loop (slu_b200_k_gemm_sub variant 30: schur_kernel_h's tile and K loop, RED epilogue into a dense
C) at K = 256 against K = 512, and the segmented K loop (variant 35) at K = 512, on the heavy levels' shapes of the bench
workload (m, n of the large nested updates).  One JSON line per shape: TFlop/s of each arm."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superlu_dist_b200 import capi  # noqa: E402


def rate(m, n, k, variant, reps=10):
    rng = np.random.default_rng(0)
    a, b, c = rng.standard_normal((m, k)), rng.standard_normal((k, n)), np.zeros((m, n))
    os.environ["SLU_B200_GEMM_VARIANT"] = str(variant)
    try:
        _, ms = capi.k_gemm_sub(a, b, c, reps=reps)
    finally:
        os.environ.pop("SLU_B200_GEMM_VARIANT", None)
    return 2.0 * m * n * k / (ms * 1e-3) / 1e12, ms


for m, n in [(4096, 4096), (8192, 8192), (12288, 6144)]:
    r256, t256 = rate(m, n, 256, 30)
    r512, t512 = rate(m, n, 512, 30)
    s512, u512 = rate(m, n, 512, 35)
    print(json.dumps({"m": m, "n": n, "tflops_k256": round(r256, 2), "tflops_k512": round(r512, 2),
                      "tflops_k512_segmented": round(s512, 2), "ms_2x_k256": round(2 * t256, 3), "ms_k512": round(t512, 3),
                      "ms_k512_segmented": round(u512, 3)}), flush=True)
