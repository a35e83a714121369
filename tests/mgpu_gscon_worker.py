"""Worker of tests/test_gpu_gscon.py (one process per GPU, launched by torch.distributed.run): the condition estimate on
the resident factors of a 1 x 1 x Pz grid (slu_b200_gscon, slu_b200_z_gscon) against a single-process handle of the same
matrix.  Every rank must take the same decisions: the same rcond and the same number of solves."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from superlu_dist_b200 import capi  # noqa: E402
from mgpu_tsolve_worker import KW, real_problem  # noqa: E402
from util import complex_problem  # noqa: E402


def estimates(prob, rank, **opt):
    h = capi.Handle(prob, rank, **opt)
    h.upload()
    assert h.factor() == 0
    out = {}
    for norm in ("1", "I"):
        rc = h.rcond(1.0, norm)
        out[norm] = (rc, h.stats().reserved[7])
    h.close()
    return out


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    err = 0.0
    for make in (real_problem, lambda **kw: complex_problem(**KW, **kw)):
        want = estimates(make(), 0, device=local)
        box = [capi.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        got = estimates(make(npdep=world, layers=[rank]), rank, device=local, world_size=world, world_rank=rank, nccl_id=box[0])
        for norm, (rc, rounds) in got.items():
            assert rounds == want[norm][1], (norm, rounds, want[norm])
            err = max(err, abs(rc - want[norm][0]) / want[norm][0])
        ranks = [None] * world
        dist.all_gather_object(ranks, got)
        assert all(r == got for r in ranks), ranks             # the same decisions and the same result on every rank
    assert err < 1e-12, err
    print(f"rank {rank}/{world}: rcond err {err:.2e}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
