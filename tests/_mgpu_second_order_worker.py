"""Multi-GPU worker for second derivatives (one process per GPU, torchrun + NCCL for the bootstrap only).  On every rank:
transpose_entries_async forward then set_values on the transpose gives the multiply bits of transpose_values, and reverse after
forward (and forward after reverse) gives back random entry vectors bit for bit; multiply_values_async with the handle's own
values equals multiply_async bit for bit; the Hessian-vector product in b of a solve agrees with the dense one of the global
matrix within 1e-9 relative (rank sums change the order)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from _mgpu_transpose_worker import _bits, _global_csr, _perturbed


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=1e-14, max_iter=3000, mega=1, resident=0, cache=1)
    for kind, g, p0 in [("convdiff", 24, 1.5), ("stencil15", 10, 14.0)]:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        dm = B.DeviceMatrix(blk)
        mt = dm._adjoint()
        rng = np.random.default_rng(21 + rank)
        dv = _cuda(_perturbed(blk.diag_arrays()[0].copy(), 2 + rank))
        ov = _cuda(_perturbed(blk.offd_arrays()[0].copy(), 5 + rank)) if blk.offd.nz else None
        dm.set_values_async(dv, ov)
        x = _cuda(rng.standard_normal((3, nloc)))
        # entry permutation: forward -> set_values equals the refresh, and exact round trips
        mt.transpose_values_async(dm)
        want = torch.empty_like(x)
        mt.multiply_async(x, want)
        pd, po = mt.transpose_entries_async(dm, dv, ov)
        mt.set_values_async(pd, po)
        got = torch.empty_like(x)
        mt.multiply_async(x, got)
        rd = _cuda(rng.standard_normal(int(blk.diag.nz)))
        ro = _cuda(rng.standard_normal(int(blk.offd.nz))) if ov is not None else None
        fd, fo = mt.transpose_entries_async(dm, rd, ro)
        bd, bo = mt.transpose_entries_async(dm, fd, fo, reverse=True)
        # an independent vector in mt's block order: forward after reverse gives it back
        td = _cuda(rng.standard_normal(int(mt.blk.diag.nz)))
        to = _cuda(rng.standard_normal(int(mt.blk.offd.nz))) if fo is not None else None
        sd, so = mt.transpose_entries_async(dm, td, to, reverse=True)
        f2d, f2o = mt.transpose_entries_async(dm, sd, so)
        torch.cuda.synchronize()
        assert _bits(got) == _bits(want), (kind, rank, "forward")
        assert _bits(bd) == _bits(rd) and (ro is None or _bits(bo) == _bits(ro)), (kind, rank, "reverse")
        assert _bits(f2d) == _bits(td) and (to is None or _bits(f2o) == _bits(to)), (kind, rank, "forward after reverse")
        # weighted multiply with the handle's own values
        for alpha, beta in ((1.0, 0.0), (-0.75, 1.0)):
            y0 = rng.standard_normal((3, nloc))
            want, got = _cuda(y0), _cuda(y0)
            dm.multiply_async(x, want, alpha=alpha, beta=beta)
            dm.multiply_values_async(dv, ov, x, got, alpha=alpha, beta=beta)
            torch.cuda.synchronize()
            assert _bits(got) == _bits(want), (kind, rank, alpha, beta)
        # HVP in b of a solve against the dense global one
        ptr, col, val = _global_csr(kind, g, p0, world, k=2)
        rows = np.repeat(np.arange(n), np.diff(ptr))
        A = torch.zeros((n, n), dtype=torch.float64).index_put((torch.from_numpy(rows), torch.from_numpy(np.asarray(col))),
                                                                torch.from_numpy(np.asarray(val)), accumulate=True).cuda()
        grng = np.random.default_rng(99)
        bg, wg, vg = (_cuda(grng.standard_normal(n)) for _ in range(3))
        sl = slice(lo, lo + nloc)

        def loss(x_, w_):
            return (w_ * x_).sum() + 0.5 * (x_ * x_).sum()
        _, hv = torch.autograd.functional.hvp(lambda bb: loss(B.solve_autograd(dm, bb), wg[sl].contiguous()),
                                              bg[sl].contiguous(), vg[sl].contiguous())
        _, hd = torch.autograd.functional.hvp(lambda bb: loss(torch.linalg.solve(A, bb), wg), bg, vg)
        rel = float((hv - hd[sl]).abs().max() / hd.abs().max())
        assert rel <= 1e-9, (kind, rank, rel)
        dm.destroy()
        if rank == 0:
            print(f"[mgpu {world}] {kind:10s} second order: entries exact, weighted multiply bit-identical, hvp {rel:.1e}",
                  flush=True)
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SECOND_ORDER_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
