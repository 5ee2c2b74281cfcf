"""Multi-GPU worker for the differentiable shifted solve (one process per GPU, torchrun + NCCL for the bootstrap only).  On every
rank: X, b.grad, diag and offd value gradients of shifted_solve_autograd are this rank's rows of the dense computation of the
whole matrix (within 1e-9 relative); sigma.grad is bit-identical on every rank and within 1e-9 of dense; dots_async gives every
rank the same bits; prepare_shifted_autograd succeeds on every rank."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from _mgpu_autograd_worker import _bits, _gather

SIGMA = np.array([0.0, 0.5, 1.25, -0.125])


def _same_on_every_rank(t, what):
    outs = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(outs, t.contiguous())
    assert all(_bits(o) == _bits(t) for o in outs), what


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=1e-14, max_iter=3000, shift_tol=1e-14, shift_max_iter=3000, mega=1, resident=0, cache=1)
    L = SIGMA.size
    for kind, g, p0 in [("convdiff", 24, 2.0), ("stencil15", 8, 14.0)]:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        dv, dc, dp = (np.asarray(a).copy() for a in blk.diag_arrays())
        ov, oc, op_ = (np.asarray(a).copy() for a in blk.offd_arrays())
        dm = B.DeviceMatrix(blk)
        dm.prepare_shifted_autograd("shifted_lopbicgstab", L)
        rng = np.random.default_rng(3 + rank)
        # ---- dots_async: every rank the same bits -----------------------------------------------------------------------
        u, v = (torch.from_numpy(rng.standard_normal((9, nloc))).cuda() for _ in range(2))
        d = dm.dots_async(u, v)
        torch.cuda.synchronize()
        _same_on_every_rank(d, (kind, "dots"))
        want = np.einsum("ji,ji->j", _gather(u.cpu().numpy()), _gather(v.cpu().numpy()))
        assert np.abs(d.cpu().numpy() - want).max() <= 1e-12 * np.abs(want).max(), (kind, rank, "dots")
        # ---- shifted_solve_autograd against dense numpy -----------------------------------------------------------------
        b, w = rng.standard_normal(nloc), rng.standard_normal((L, nloc))
        tb, tdv, tov = (torch.from_numpy(a).cuda().requires_grad_() for a in (b, dv, ov))
        ts = torch.from_numpy(SIGMA.copy()).cuda().requires_grad_()
        x = B.shifted_solve_autograd(dm, tb, ts, diag_val=tdv, offd_val=tov if ov.size else None)
        (x * torch.from_numpy(w).cuda()).sum().backward()
        torch.cuda.synchronize()
        _same_on_every_rank(ts.grad, (kind, "sigma.grad"))
        ptr, col, val = (np.asarray(p) for p in B.block_to_global_csr(blk, rank=rank))
        rows_all = _gather(np.repeat(np.arange(nloc) + lo, np.diff(ptr.astype(np.int64)))[None, :].astype(np.float64))[0]
        cols_all = _gather(col[None, :].astype(np.float64))[0]
        vals_all = _gather(val[None, :])[0]
        A = np.zeros((n, n))
        np.add.at(A, (rows_all.astype(np.int64), cols_all.astype(np.int64)), vals_all)
        bg, wg = _gather(b[None, :])[0], _gather(w)
        xd = np.stack([np.linalg.solve(A + s * np.eye(n), bg) for s in SIGMA])
        lam = np.stack([np.linalg.solve(A.T + s * np.eye(n), wg[j]) for j, s in enumerate(SIGMA)])
        drows = np.repeat(np.arange(nloc), np.diff(dp.astype(np.int64)))
        orows = np.repeat(np.arange(nloc), np.diff(op_.astype(np.int64)))
        checks = [(x, xd[:, lo:lo + nloc]), (tb.grad, lam.sum(axis=0)[lo:lo + nloc]),
                  (ts.grad, -np.einsum("ji,ji->j", lam, xd)),
                  (tdv.grad, -(lam[:, drows + lo] * xd[:, dc.astype(np.int64) + lo]).sum(axis=0))]
        if ov.size:
            checks.append((tov.grad, -(lam[:, orows + lo] * xd[:, oc.astype(np.int64)]).sum(axis=0)))
        for k, (got, want) in enumerate(checks):
            got = got.detach().cpu().numpy()
            assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max(), (kind, rank, k)
        dm.destroy()
        if rank == 0:
            print(f"[mgpu {world}] {kind:10s} shifted autograd within the dense bound, sigma.grad and dots identical on every "
                  f"rank", flush=True)
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SHIFTED_AUTOGRAD_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
