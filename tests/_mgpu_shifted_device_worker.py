"""Multi-GPU worker of the shifted solvers on device vectors (one process per GPU, torchrun + NCCL for the bootstrap only): on its
row block every rank runs each of the four shifted methods through the host path (numpy) and the device path (CUDA tensors,
bicg_shifted_solve_dev), with BICG_SHIFT_ERROR=1, and requires the two to be bitwise equal.  random n = 3001 gives an odd n_loc on
at least one rank at 2 and 4 ranks; the x_set tensor of one run sits at a one-element offset inside a larger tensor."""
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
from helpers import SHIFTED_CASES
from shifted_lop_cases import shifted_lop_problem

METHODS = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _results(L, k, st):
    seed, stop = B.last_shift_info(L)
    return dict(k=k, iters=st["iters"], conv=st["converged"], res=_bits(st["final_res"]), launches=st["kernel_launches"],
                hist=_bits(B.last_history()), seed=seed, stop=stop.tolist(), err=_bits(B.last_shift_error(L)))


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1, shift_tol=1e-12, shift_max_iter=1000, shift_error=0)
    rank, world = B.comm_init_torch()
    problems = [("random3001_L13", "random", 3001, 8, 13, 0.05 / 13, 6), SHIFTED_CASES[1]]
    odd = False
    for case in problems:
        name, kind, g, p0 = case[:4]
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        odd |= nloc % 2 == 1
        ptr, col, val = B.block_to_global_csr(B.gen_block(kind, g, p0))
        sigma, bg, seed = shifted_lop_problem(O, n, ptr, col, val, case)
        L = sigma.size
        bl = np.ascontiguousarray(bg[lo:lo + nloc])
        dm = B.DeviceMatrix(blk)
        for i, method in enumerate(METHODS):
            B.set_options(shift_error=1)
            xs = np.zeros((L, nloc)); rs = bl.copy()
            host = _results(L, *dm.shifted_solve(method, xs, rs, sigma, seed))
            if i % 2:
                big = torch.zeros(L * nloc + 1, dtype=torch.float64, device="cuda")
                xt = big[1:].view(L, nloc)
            else:
                xt = torch.zeros((L, nloc), dtype=torch.float64, device="cuda")
            rt = torch.from_numpy(bl.copy()).cuda()
            p0_ = xt.data_ptr()
            k, st = dm.shifted_solve(method, xt, rt, sigma, seed)
            dev = _results(L, k, st)
            B.set_options(shift_error=0)
            assert xt.data_ptr() == p0_ and st["h2d_bytes"] == 0 and st["d2h_bytes"] == 0, (name, method, rank)
            assert dev == host, (name, method, rank, host, dev)
            assert _bits(xt.cpu().numpy()) == _bits(xs) and _bits(rt.cpu().numpy()) == _bits(rs), (name, method, rank)
            if rank == 0:
                print(f"[mgpu {world}] {name} {method}: device path = host path ({host['k']})", flush=True)
        dm.destroy()
    flag = torch.tensor([1 if odd else 0], device="cuda")
    dist.all_reduce(flag)
    assert flag.item() >= 1, "no rank had an odd n_loc"
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SHIFTED_DEVICE_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
