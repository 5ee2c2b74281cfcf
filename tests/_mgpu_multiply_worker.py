"""Multi-GPU worker for the batched multiply on a resident matrix (one process per GPU, torchrun + NCCL for the bootstrap only).
On every rank: y_j = A x_j for full, partial and several launches is bit-identical to spmv(x_j) and within 1e-13 of the oracle's
long-double global product; one 17-vector call equals 17 single-vector calls; and update values -> b = A 1 -> solve -> b - A x
enqueued on a side stream equals the synchronous sequence bit for bit."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mpi_bicgstab_b200 as B
import oracle as O


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _global_xs(nvec, n, seed):
    """the same global vectors on every rank"""
    return np.random.default_rng(seed + 31 * nvec).standard_normal((nvec, n))


def _perturbed(v, k):
    return v * (1.0 + ((np.arange(v.size) * (2 * k + 1) + k) % 7) / 64.0)


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=1e-10, max_iter=600, mega=1, resident=0, cache=1)
    for kind, g, p0 in [("stencil15", 40, 14.0), ("convdiff", 200, 1.5), ("random", 20000, 32)]:
        make = lambda: B.gen_block(kind, g, p0, rank=rank, world=world)
        blk = make()
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        dm = B.DeviceMatrix(blk)
        # the global matrix, every rank's rows in the reference's merged order, for the oracle
        parts = [B.block_to_global_csr(B.gen_block(kind, g, p0, rank=p, world=world), rank=p) for p in range(world)]
        gptr = np.concatenate([[0]] + [p[0][1:] + sum(int(q[0][-1]) for q in parts[:i]) for i, p in enumerate(parts)])
        gcol = np.concatenate([p[1] for p in parts])
        gval = np.concatenate([p[2] for p in parts])
        for nvec in (1, 3, 8, 9, 17):
            xg = _global_xs(nvec, n, 1)
            x = np.ascontiguousarray(xg[:, lo:lo + nloc])
            y = dm.multiply(x)
            ty = torch.empty(nvec, nloc, dtype=torch.float64, device="cuda")
            dm.multiply_async(torch.from_numpy(x).cuda(), ty)
            torch.cuda.synchronize()
            for j in range(nvec):
                want = dm.spmv(x[j])
                assert _bits(y[j]) == _bits(want) and _bits(ty[j]) == _bits(want), (kind, rank, nvec, j)
                y_ref = O.spmv(n, gptr, gcol, gval, xg[j], P=world, long_double=True)[lo:lo + nloc]
                assert np.abs(y[j] - y_ref).max() <= 1e-13 * np.abs(y_ref).max(), (kind, rank, nvec, j)
        # batch independence, with a shift and beta != 0
        x = torch.from_numpy(np.ascontiguousarray(_global_xs(17, n, 3)[:, lo:lo + nloc])).cuda()
        y0 = torch.from_numpy(np.ascontiguousarray(_global_xs(17, n, 4)[:, lo:lo + nloc])).cuda()
        sigma = torch.from_numpy(np.linspace(-1.0, 2.0, 17)).cuda()
        y, singles = y0.clone(), y0.clone()
        dm.multiply_async(x, y, alpha=-0.5, beta=2.0, sigma=sigma)
        for j in range(17):
            dm.multiply_async(x[j], singles[j], alpha=-0.5, beta=2.0, sigma=sigma[j:j + 1])
        torch.cuda.synchronize()
        assert _bits(y) == _bits(singles), (kind, rank)
        # stream order: update values, b = A 1, solve, b - A x
        dv, ov = blk.diag_arrays()[0].copy(), blk.offd_arrays()[0].copy()
        dv2, ov2 = _perturbed(dv, 2 + rank), _perturbed(ov, 5 + rank)
        dm.set_values(dv2, ov2)
        b = dm.multiply(np.ones(nloc))
        xs, r = np.zeros(nloc), b.copy()
        it, _ = dm.solve("bicgstab", xs, r)
        res = dm.multiply(xs, b.copy(), alpha=-1.0, beta=1.0)
        want = [_bits(b), _bits(xs), _bits(r), _bits(res), it]
        dm.set_values(dv, ov)
        dm.prepare_async("bicgstab")
        tv, to = torch.from_numpy(dv2).cuda(), torch.from_numpy(ov2).cuda()
        t1, tb, tx, tr, tres = (torch.ones(nloc, dtype=torch.float64, device="cuda"),
                                *(torch.empty(nloc, dtype=torch.float64, device="cuda") for _ in range(4)))
        result = torch.zeros(24, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            dm.set_values_async(tv, to)
            dm.multiply_async(t1, tb)
            tx.zero_()
            tr.copy_(tb)
            dm.solve_async("bicgstab", tx, tr, result=result)
            tres.copy_(tb)
            dm.multiply_async(tx, tres, alpha=-1.0, beta=1.0)
        s.synchronize()
        got = [_bits(tb), _bits(tx), _bits(tr), _bits(tres), B.decode_result(result)["iters"]]
        assert got == want, (kind, rank)
        dm.destroy()
        if rank == 0:
            print(f"[mgpu {world}] {kind:10s} multiply: bit-identical to spmv, batch-independent, stream-ordered", flush=True)
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_MULTIPLY_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
