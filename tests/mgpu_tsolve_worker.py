"""Worker of tests/test_gpu_solve_trans.py (one process per GPU, launched by torch.distributed.run): the transposed and
conjugate-transposed solves on the resident factors of a 1 x 1 x Pz grid (slu_b200_solve_trans, slu_b200_z_solve_trans),
against a single-process handle of the same matrix.  Every rank builds the same b from a fixed seed and must receive the
full solution."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from superlu_dist_b200 import capi  # noqa: E402
from test_gpu_solve_trans import unsym_values  # noqa: E402
from util import complex_problem, poisson_problem  # noqa: E402

KW = dict(N=12, leaf=8, relax=16, maxsup=64)


def real_problem(**kw):
    prob, (rp, ci, v) = poisson_problem(**KW, **kw)
    for z in prob.layers:
        prob.fill_layer(z, rp, ci, unsym_values(rp, ci, v))
    return prob


def solves(prob, rank, b, transes, **opt):
    h = capi.Handle(prob, rank, **opt)
    h.upload()
    assert h.factor() == 0
    out = {t: (h.solve(b, trans=t), h.solve(b[1], trans=t)) for t in transes}
    h.close()
    return out


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    rng = np.random.default_rng(7)
    err = 0.0
    for make, transes, cplx in ((real_problem, ("T",), False), (lambda **kw: complex_problem(**KW, **kw), ("T", "H"), True)):
        one = make()
        b = rng.standard_normal((2, one.n)) + (1j * rng.standard_normal((2, one.n)) if cplx else 0)
        want = solves(one, 0, b, transes, device=local)
        box = [capi.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        got = solves(make(npdep=world, layers=[rank]), rank, b, transes, device=local, world_size=world, world_rank=rank,
                     nccl_id=box[0])
        for t in transes:
            for g, w in zip(got[t], want[t]):
                err = max(err, float(np.abs(g - w).max() / np.abs(w).max()))
    assert err < 1e-12, err
    print(f"rank {rank}/{world}: transposed solve err {err:.2e}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
