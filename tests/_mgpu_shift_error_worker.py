"""Multi-GPU worker of the shifted-solution check (one process per GPU, torchrun + NCCL for the bootstrap only): on its row block
every rank runs bicg_shift_residuals (host and device vectors) and two shifted solves with BICG_SHIFT_ERROR=1; the errors, the same
on every rank, must match the exact P = 1 evaluation of the gathered x_j, and only rank 0 prints the error block."""
import math
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
import oracle as O
from shifted_lop_cases import SHIFTED_LOP_CASES, shifted_lop_problem
from test_gpu_shift_error import exact_errors


def _captured(fn):
    """Run fn() with this process's fd 1 redirected to a file; returns (fn's result, what was written there)."""
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(f.fileno(), 1)
        try:
            res = fn()
            B.lib.bicg_synchronize()
            import ctypes
            ctypes.CDLL(None).fflush(None)
        finally:
            os.dup2(saved, 1)
            os.close(saved)
        f.seek(0)
        return res, f.read()


def _same_everywhere(v):
    t = torch.tensor(np.nan_to_num(np.asarray(v, dtype=np.float64), nan=-1.0), device="cuda")
    lo, hi = t.clone(), t.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    return torch.equal(lo, hi)


def _gather(x_loc, world):
    t = torch.from_numpy(np.ascontiguousarray(x_loc)).cuda()
    parts = [None] * world
    dist.all_gather_object(parts, t.cpu().numpy())
    return np.concatenate(parts, axis=-1)


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1, shift_tol=1e-12, shift_max_iter=1000, shift_error=0)
    rank, world = B.comm_init_torch()
    for kind, g, p0 in (("stencil15", 12, 14.0), ("random", 3001, 32)):
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        ptr, col, val = B.block_to_global_csr(B.gen_block(kind, g, p0))
        dm = B.DeviceMatrix(blk)
        for L in (1, 13):                                   # 13: one full batch of 8 halo slots and a remainder
            rng = np.random.default_rng(L)
            x = rng.standard_normal((L, n)); b = rng.standard_normal(n); sigma = rng.uniform(-0.5, 0.5, L)
            want, _ = exact_errors(ptr, col, val, x, b, sigma)
            xl, bl = np.ascontiguousarray(x[:, lo:lo + nloc]), np.ascontiguousarray(b[lo:lo + nloc])
            got_h = dm.shift_residuals(xl, bl, sigma)
            got_d = dm.shift_residuals(torch.from_numpy(xl).cuda(), torch.from_numpy(bl).cuda(), sigma)
            for got in (got_h, got_d):
                assert np.all(np.abs(got - want) <= 1e-13 * want), (kind, L, rank, got, want)
            assert np.array_equal(got_h, got_d) and _same_everywhere(got_h)
        dm.destroy()
    B.set_options(quiet=0)
    for case in (SHIFTED_LOP_CASES[0], SHIFTED_LOP_CASES[1]):
        name, kind, g, p0 = case[:4]
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        ptr, col, val = B.block_to_global_csr(B.gen_block(kind, g, p0))
        sigma, bg, seed = shifted_lop_problem(O, n, ptr, col, val, case)
        dm = B.DeviceMatrix(blk)
        for method in ("shifted_lopbicg_switching", "shifted_lopbicgstab"):
            B.set_options(shift_error=1)
            xs = np.zeros((sigma.size, nloc)); rs = np.ascontiguousarray(bg[lo:lo + nloc])
            _, out = _captured(lambda: dm.shifted_solve(method, xs, rs, sigma, seed))
            B.set_options(shift_error=0)
            err = B.last_shift_error(sigma.size)
            assert err.size == sigma.size and _same_everywhere(err), (name, method, rank)
            assert out.count("seed(0:seed, 1:shift), sigma, relative error\n") == (1 if rank == 0 else 0), (rank, out)
            assert out.count("Total time") == (1 if rank == 0 else 0), (rank, out)
            xg = _gather(xs, world)
            want, scale = exact_errors(ptr, col, val, xg, bg, sigma)
            fin = np.isfinite(want)
            assert np.array_equal(fin, np.isfinite(err))
            assert np.all(np.abs(err[fin] - want[fin]) <= 1e-13 * scale[fin]), (name, method, rank, err, want)
            if rank == 0:
                print(f"[mgpu {world}] {name} {method}: max error {np.nanmax(err):.3e}", flush=True)
        dm.destroy()
    B.set_options(quiet=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SHIFT_ERROR_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
