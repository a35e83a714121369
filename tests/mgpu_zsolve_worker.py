"""Worker of tests/test_gpu_solve_complex.py (one process per GPU, launched by torch.distributed.run): the doublecomplex
solve on the resident factors of a 1 x 1 x Pz grid (slu_b200_z_solve).  Every rank builds the same b from a fixed seed
and must receive the full solution."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from superlu_dist_b200 import capi  # noqa: E402
from util import complex_problem  # noqa: E402

KW = dict(N=12, leaf=8, relax=16, maxsup=64)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    one = complex_problem(**KW)
    A = one.dense(one.layers[0], False)
    rng = np.random.default_rng(7)
    xtrue = rng.standard_normal((2, one.n)) + 1j * rng.standard_normal((2, one.n))
    b = (A @ xtrue.T).T
    box = [capi.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    prob = complex_problem(npdep=world, layers=[rank], **KW)
    h = capi.Handle(prob, rank, device=local, world_size=world, world_rank=rank, nccl_id=box[0])
    h.upload()
    assert h.factor() == 0
    x = h.solve(b)
    x1 = h.solve(b[1])
    h.close()
    err = max(float(np.abs(x - xtrue).max()), float(np.abs(x1 - xtrue[1]).max())) / float(np.abs(xtrue).max())
    assert err < 1e-10, err
    print(f"rank {rank}/{world}: complex solve err {err:.2e}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
