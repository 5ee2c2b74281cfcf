"""Multi-GPU worker of shifted_lopbicg (one process per GPU, torchrun + NCCL for the bootstrap only): every rank runs the fixed-seed
solve collectively on its row block and checks its slice of every x_j, the iteration count and the stop iterations against the
oracle's P-rank emulation (same partition, same diag-then-offd association, dots summed in rank order), on a case without a seed
switch and on one whose seed converges first and keeps iterating."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
import oracle as O
import shifted_fixed_oracle as OF
from helpers import SHIFTED_CASES


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1, shift_tol=1e-12, shift_max_iter=1000)
    rank, world = B.comm_init_torch()
    for case in (SHIFTED_CASES[0], SHIFTED_CASES[1]):
        name, kind, g, p0, L, scale, seed = case
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        ptr, col, val = B.block_to_global_csr(B.gen_block(kind, g, p0))
        sigma = (np.arange(L) + 1) * scale
        bg = O.spmv(n, ptr, col, val, np.ones(n), P=world)
        O.daxpy(sigma[seed], np.ones(n), bg)
        ref = OF.shifted_fixed_solve(n, ptr, col, val, bg, sigma, seed, P=world, tol=1e-12, max_iter=1000)
        xs = np.zeros((L, nloc)); rs = np.ascontiguousarray(bg[lo:lo + nloc])
        ret = B.shifted_lopbicg(blk, xs, rs, sigma, seed)
        hist = B.last_history()
        end_seed, stop = B.last_shift_info(L)
        assert abs(ret - ref["ret"]) <= 2, (name, ret, ref["ret"])
        assert end_seed == seed and np.all(np.abs(stop - ref["stop_iter"]) <= 2), (name, stop, ref["stop_iter"])
        m = min(10, ret, ref["ret"])
        got, want = np.sqrt(hist[1:m + 1]), np.sqrt(ref["hist"][1:m + 1])
        assert np.all(np.abs(got - want) <= 1e-10 * want + 1e-15), (name, rank, got, want)
        for j in range(L):
            assert np.abs(xs[j] - ref["x"][j][lo:lo + nloc]).max() <= 1e-8 * np.abs(ref["x"][j]).max(), (name, j, rank)
        # every rank ran the same number of iterations and saw the same residual
        t = torch.tensor([float(ret), float(hist[min(m, ret)])], dtype=torch.float64, device="cuda")
        tmax, tmin = t.clone(), t.clone()
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX); dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
        assert torch.equal(tmax, tmin), "ranks disagree on iteration count / residual"
        if rank == 0:
            print(f"[mgpu {world}] {name} shifted_lopbicg: {ret} it (oracle {ref['ret']}), seed stopped at {stop[seed]}", flush=True)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SHIFTED_FIXED_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
