"""The int8 tensor-core path (slu_ozaki.cu): int8-slice GEMM on wgmma (s8 x s8 -> s32) with register accumulators.

Tolerances.  With S slices an operand row is known to 2^-(7S-1) of ITS power-of-two scale 2^e (max|row| <= 2^e < 2 max|row|),
and the S cross terms of weight 2^-(7S+5) per (s, t) pair with s + t = S are dropped, so for every element
    |(C - A B)_ij - exact| <= k * (S + 2) * 2^(4-7S) * rowmax_i * colmax_j        (worst case, any data)
= k * 2.9e-11 (S = 6), 2.6e-13 (S = 7), 2.2e-15 (S = 8) in units of rowmax * colmax.  The path is opt-in (tc_slices).  Typical data sit one to two
orders below; the worst case is approached
only for k of a few (no averaging).  Inside the factorization the parity bar of the other tests applies unchanged: entry-wise
1e-10 relative to max|factor| against the oracle, residual probe <= 1e-12."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle
from superlu_dist_b200 import capi
from util import poisson_problem, rel_err, residual_probe

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
BOUND = {6: 3e-11, 7: 3e-13, 8: 5e-15}       # the worst-case bound above (S = 8: plus the rounding of the NumPy reference)


def _gemm_child(variant):
    """slu_b200_k_gemm_sub reads SLU_B200_GEMM_VARIANT per call, but a trap in a tensor-core kernel would poison this
    process's CUDA context: run the kernel-level cases in a child."""
    code = f'''
import os, sys, json
import numpy as np
sys.path.insert(0, {os.path.dirname(HERE)!r})
from superlu_dist_b200 import capi
os.environ["SLU_B200_GEMM_VARIANT"] = "{variant}"
rng = np.random.default_rng(7)
worst = 0.0
for (m, n, k) in [(1, 1, 1), (7, 5, 3), (128, 32, 32), (130, 70, 100), (300, 200, 256), (513, 129, 37), (257, 95, 416), (640, 320, 512)]:
    a = rng.standard_normal((m, k)) * np.exp(rng.uniform(-6, 6, (m, 1)))     # rows / columns of very different scale
    b = rng.standard_normal((k, n)) * np.exp(rng.uniform(-6, 6, (1, n)))
    a[m // 2, :] = 0.0                                                       # an all-zero row
    c = rng.standard_normal((m, n))
    out, _ = capi.k_gemm_sub(a, b, c)
    ref = c - a @ b
    bound = k * np.maximum(np.abs(a).max(axis=1), 1e-300)[:, None] * np.abs(b).max(axis=0)[None, :]
    # the final c + (-ab) rounds at eps * |c| on both sides (NumPy and the RED.ADD): not part of the product's error
    excess = np.maximum(np.abs(out - ref) - 4.5e-16 * np.abs(ref), 0.0)
    worst = max(worst, float((excess / np.maximum(bound, 1e-300)).max()))
print(json.dumps({{"worst": worst}}))
'''
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    import json
    return json.loads(r.stdout.strip().splitlines()[-1])["worst"]


@pytest.mark.parametrize("variant,slices", [(120, 6), (130, 7), (140, 8), (131, 7)])
def test_tcgen05_gemm_against_numpy(variant, slices):
    """C -= A B through the int8 slices (one tile per CTA, 2 stages: 120/130/140; 3 stages: 131) against NumPy, rows and
    columns spanning 5 orders of magnitude.  (The cluster-multicast variants 132-134 are benchmark-only: slower.)"""
    worst = _gemm_child(variant)
    assert worst <= BOUND[slices], (variant, worst)


_K1, _K2 = dict(N=14, leaf=8, relax=16, maxsup=256), dict(N=18, leaf=16, relax=32, maxsup=256)
_K3, _K4 = dict(N=8, leaf=4, relax=8, maxsup=200, fem=3), dict(N=20, leaf=32, relax=64, maxsup=400)


@pytest.mark.parametrize("kw,slices", [(_K1, 7), (_K2, 7), (_K3, 7), (_K4, 7), (_K2, 6), (_K2, 8), (_K4, 8)])
def test_factorization_through_tcgen05(kw, slices):
    """Whole pdgstrf3d with the wide supernodes (>= 64 columns here) on the int8 tensor-core path against the oracle: same bar as
    the FP64 path.  maxsup = 400 exercises more than 8 k-steps (no int32 pair recombination)."""
    prob, _ = poisson_problem(**kw)
    chk, _ = poisson_problem(**kw)
    info, st = capi.pdgstrf3d(prob, 0, tc_slices=slices, tc_min_ns=64)
    oinfo, oops, _ = oracle.factor(chk)
    assert info == oinfo == 0
    assert st.reserved[1] > 0 and int(st.reserved[3]) == slices          # the path was taken
    assert abs(st.ops_fact - oops) <= 1e-9 * oops
    a, b = prob.layers[0], chk.layers[0]
    assert rel_err(a.lval, b.lval) < 1e-10 and rel_err(a.uval, b.uval) < 1e-10


def test_tcgen05_default_off_and_opt_in_residual():
    """The path is off by default (its error is relative to rowmax * colmax of each update, so it needs balanced pivot
    scales: tests/test_scaled_parity.py) and with options.reserved[4] = -1 (FP64 DMMA only); opted in with 7 slices it
    carries most of the Schur flops and the size-independent residual probe stays at the 1e-15 level."""
    for tc in (0, -1):
        prob, _ = poisson_problem(32, leaf=64, relax=32, maxsup=256)
        pre = prob.layers[0].copy()
        every = np.ones(prob.nsupers, bool)
        info, st = capi.pdgstrf3d(prob, 0, tc_slices=tc)
        assert info == 0 and st.reserved[1] == 0 and int(st.reserved[3]) == 0, tc
        assert residual_probe(prob, [(pre, every)], [(prob.layers[0], every)]) < 1e-12
    prob2, _ = poisson_problem(32, leaf=64, relax=32, maxsup=256)
    info, st = capi.pdgstrf3d(prob2, 0, tc_slices=7)
    assert info == 0 and st.reserved[1] > 0.5 * st.ops_schur and int(st.reserved[3]) == 7   # on: most of the flops
    assert residual_probe(prob2, [(pre, every)], [(prob2.layers[0], every)]) < 1e-12
