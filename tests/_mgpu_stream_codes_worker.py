"""Multi-GPU worker for the 16-bit column codes of the persistent kernel (one process per GPU, torchrun + NCCL for the
bootstrap only).  With several ranks a CTA's columns are own columns and ghost slots; both windows share its 16-bit codes.
Every rank checks that a coded solve and a solve forced to 32-bit columns agree bit for bit on its slice."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from helpers import METHODS, RR

TOL = 1e-10


def _run(dm, method, nloc, codes):
    dm.stream_codes(codes)
    r = dm.spmv(np.ones(nloc))
    x = np.zeros(nloc)
    kw = RR if method.endswith("rr") else {}
    it, st = dm.solve(method, x, r, **kw)
    assert st["kernel_launches"] <= 8, ("not the persistent kernel", method)
    return it, x, r, B.last_history(), dm.coded_ctas()


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=TOL, max_iter=600, mega=1, resident=0, cache=1)
    for kind, g, p0 in [("stencil15", 40, 14.0), ("convdiff", 200, 1.5), ("laplace5", 300, 0.0)]:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        dm = B.DeviceMatrix(blk)
        for method in METHODS:
            it1, x1, r1, h1, n1 = _run(dm, method, blk.n_loc, True)
            it0, x0, r0, h0, n0 = _run(dm, method, blk.n_loc, False)
            assert n1 > 0 and n0 == 0, (kind, method, rank, n1, n0)
            assert it1 == it0 and np.array_equal(h1, h0), (kind, method, rank, it1, it0)
            assert np.array_equal(x1, x0) and np.array_equal(r1, r0), (kind, method, rank)
            assert np.abs(x1 - 1).max() < 1e-6, (kind, method, rank)
            if rank == 0:
                print(f"[mgpu {world}] {kind:10s} {method:17s} {it1:4d} it, coded CTAs {n1}: bit-identical to 32-bit columns", flush=True)
        dm.destroy()
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_STREAM_CODES_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
