"""Multi-GPU worker for the value gradient and the differentiable solve (one process per GPU, torchrun + NCCL for the bootstrap
only).  On every rank: value_grad's diag and offd outputs equal the replica on the gathered column vectors bit for bit (ghost
columns come through the halo), in the order of this rank's blocks; the gradients of solve_autograd agree with dense numpy; a
captured forward + backward replays bit-identically to eager runs; values without the offd part are refused."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from test_gpu_value_grad import replica


def _bits(a):
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _gather(a):
    """the rows of every rank, concatenated in rank order (a: this rank's (k, n_loc) block)"""
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    sizes = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(dist.get_world_size())]
    dist.all_gather(sizes, torch.tensor([t.shape[-1]], device="cuda"))
    m = int(max(s.item() for s in sizes))
    pad = torch.zeros(t.shape[0], m, dtype=torch.float64, device="cuda")
    pad[:, :t.shape[-1]] = t
    outs = [torch.empty_like(pad) for _ in sizes]
    dist.all_gather(outs, pad)
    return np.concatenate([o[:, :int(s.item())].cpu().numpy() for o, s in zip(outs, sizes)], axis=1)


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=1e-14, max_iter=3000, mega=1, resident=0, cache=1)
    for kind, g, p0 in [("convdiff", 24, 2.0), ("random", 3000, 12)]:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        dv, dc, dp = (np.asarray(a).copy() for a in blk.diag_arrays())
        ov, oc, op_ = (np.asarray(a).copy() for a in blk.offd_arrays())
        dm = B.DeviceMatrix(blk)
        rng = np.random.default_rng(3 + rank)
        # ---- value_grad against the replica on the gathered v (9 vectors: two batches) ------------------------------------
        u, v = rng.standard_normal((9, nloc)), rng.standard_normal((9, nloc))
        vg = _gather(v)
        gd, go = dm.value_grad(u, v, alpha=-1.0)
        drows = np.repeat(np.arange(nloc), np.diff(dp.astype(np.int64)))
        orows = np.repeat(np.arange(nloc), np.diff(op_.astype(np.int64)))
        assert _bits(gd) == _bits(replica(drows, dc.astype(np.int64) + lo, u, vg, -1.0, 0.0, None)), (kind, rank, "diag")
        if ov.size:
            assert go is not None and _bits(go) == _bits(replica(orows, oc.astype(np.int64), u, vg, -1.0, 0.0, None)), (kind, rank)
        tg = dm.value_grad_async(torch.from_numpy(u).cuda(), torch.from_numpy(v).cuda(), alpha=-1.0)
        torch.cuda.synchronize()
        assert _bits(tg[0]) == _bits(gd) and (go is None or _bits(tg[1]) == _bits(go)), (kind, rank, "async")
        # ---- solve_autograd against dense numpy -------------------------------------------------------------------------
        b, w = rng.standard_normal(nloc), rng.standard_normal(nloc)
        tb, tdv, tov = (torch.from_numpy(a).cuda().requires_grad_() for a in (b, dv, ov))
        x = B.solve_autograd(dm, tb, diag_val=tdv, offd_val=tov if ov.size else None)
        (x * torch.from_numpy(w).cuda()).sum().backward()
        ptr, col, val = B.block_to_global_csr(blk, rank=rank)
        parts = [np.asarray(p) for p in (ptr, col, val)]
        rows_all = _gather(np.repeat(np.arange(nloc) + lo, np.diff(parts[0].astype(np.int64)))[None, :].astype(np.float64))[0]
        cols_all = _gather(parts[1][None, :].astype(np.float64))[0]
        vals_all = _gather(parts[2][None, :])[0]
        A = np.zeros((n, n))
        np.add.at(A, (rows_all.astype(np.int64), cols_all.astype(np.int64)), vals_all)
        xd = np.linalg.solve(A, _gather(b[None, :])[0])
        lam = np.linalg.solve(A.T, _gather(w[None, :])[0])
        for got, want in ((x, xd[lo:lo + nloc]), (tb.grad, lam[lo:lo + nloc]),
                          (tdv.grad, -lam[drows + lo] * xd[dc.astype(np.int64) + lo])):
            got = got.detach().cpu().numpy()
            assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max(), (kind, rank)
        if ov.size:
            want = -lam[orows + lo] * xd[oc.astype(np.int64)]
            assert np.abs(tov.grad.cpu().numpy() - want).max() <= 1e-9 * np.abs(want).max(), (kind, rank)
            try:
                B.solve_autograd(dm, tb.detach(), diag_val=tdv.detach())
                raise AssertionError("values without offd_val were accepted")
            except ValueError:
                pass
        # ---- a captured forward + backward replays on every rank ---------------------------------------------------------
        dm.prepare_autograd("bicgstab")
        cb, cv, co = (torch.from_numpy(a.copy()).cuda().requires_grad_() for a in (b, dv, ov))
        tw = torch.from_numpy(w).cuda()
        kw = dict(offd_val=co) if ov.size else {}
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            xw = B.solve_autograd(dm, cb, diag_val=cv, **kw)
            (xw * tw).sum().backward()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        cb.grad = cv.grad = co.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            xs = B.solve_autograd(dm, cb, diag_val=cv, **kw)
            (xs * tw).sum().backward()
        for k in (1, 2):
            bk = rng.standard_normal(nloc)
            dk = dv * (1.0 + k / 64.0)
            with torch.no_grad():
                cb.copy_(torch.from_numpy(bk))
                cv.copy_(torch.from_numpy(dk))
            graph.replay()
            torch.cuda.synchronize()
            eb, ed, eo = (torch.from_numpy(a).cuda().requires_grad_() for a in (bk, dk, ov))
            xe = B.solve_autograd(dm, eb, diag_val=ed, **(dict(offd_val=eo) if ov.size else {}))
            (xe * tw).sum().backward()
            torch.cuda.synchronize()
            assert [_bits(xs), _bits(cb.grad), _bits(cv.grad)] == [_bits(xe), _bits(eb.grad), _bits(ed.grad)], (kind, rank, k)
        del graph
        dm.destroy()
        if rank == 0:
            print(f"[mgpu {world}] {kind:10s} value gradient bit-identical to the replica, autograd within the dense bound, "
                  f"captured backward replays", flush=True)
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_AUTOGRAD_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
