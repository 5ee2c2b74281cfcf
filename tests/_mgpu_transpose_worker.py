"""Multi-GPU worker for the transpose of a resident matrix (one process per GPU, torchrun + NCCL for the bootstrap only).  On
every rank: the transpose's spmv, batched multiply and solve are bit-identical to those of a handle created from this rank's
blocks of the stably transposed global CSR, and its product is within rounding of scipy's A^T x; after an update of the
source's values, set_values_async -> transpose_values_async -> multiply_async / solve_async on a side stream equals a fresh
transpose of the new values."""
import os
import sys

import numpy as np
import scipy.sparse as sp
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from test_gpu_transpose import transposed_csr


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _perturbed(v, k):
    return v * (1.0 + ((np.arange(v.size) * (2 * k + 1) + k) % 7) / 64.0)


def _global_csr(kind, g, p0, world, k=None):
    """The global CSR of A, every rank's rows in the merged order; k: every rank's values perturbed (diag by k + rank, offd by
    k + 3 + rank), as that rank sets them."""
    parts = []
    for p in range(world):
        blk = B.gen_block(kind, g, p0, rank=p, world=world)
        if k is not None:
            blk.diag_arrays()[0][:] = _perturbed(blk.diag_arrays()[0].copy(), k + p)
            if blk.offd.nz:
                blk.offd_arrays()[0][:] = _perturbed(blk.offd_arrays()[0].copy(), k + 3 + p)
        parts.append(B.block_to_global_csr(blk, rank=p))
    ptr = np.concatenate([[0]] + [pp[0][1:] + sum(int(q[0][-1]) for q in parts[:i]) for i, pp in enumerate(parts)])
    return ptr.astype(np.int64), np.concatenate([pp[1] for pp in parts]), np.concatenate([pp[2] for pp in parts])


def _check(dm_t, fresh, A, n, nloc, lo, what):
    rng = np.random.default_rng(11)
    xg = rng.standard_normal((3, n))
    x = np.ascontiguousarray(xg[:, lo:lo + nloc])
    y, want = dm_t.multiply(x), fresh.multiply(x)
    assert _bits(y) == _bits(want), what
    assert _bits(dm_t.spmv(x[0])) == _bits(fresh.spmv(x[0])), what
    ref = (A.T @ xg.T).T[:, lo:lo + nloc]
    scale = (abs(A).T @ abs(xg).T).T[:, lo:lo + nloc]
    assert np.all(np.abs(y - ref) <= 1e-14 * scale), what
    b = fresh.multiply(np.ones(nloc))
    got, exp = [], []
    for dm, out in ((dm_t, got), (fresh, exp)):
        xs, r = np.zeros(nloc), b.copy()
        it, _ = dm.solve("bicgstab", xs, r)
        out += [it, _bits(xs), _bits(r), _bits(B.last_history())]
    assert got == exp, what


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=1e-10, max_iter=600, mega=1, resident=0, cache=1)
    for kind, g, p0 in [("convdiff", 120, 1.5), ("random", 20000, 12), ("stencil15", 30, 14.0)]:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
        dm = B.DeviceMatrix(blk)
        mt = dm.transpose()
        ptr, col, val = _global_csr(kind, g, p0, world)
        tp, tc, tv = transposed_csr(n, ptr, col, val)
        fresh = B.DeviceMatrix(B.blocks_from_csr(n, tp, tc, tv, rank=rank, world=world))
        A = sp.csr_matrix((val, col, ptr), shape=(n, n))
        _check(mt, fresh, A, n, nloc, lo, (kind, rank, "created"))
        fresh.destroy()
        # update the source's values, then refresh the transpose and use it, all on a side stream
        dv2 = _perturbed(blk.diag_arrays()[0].copy(), 2 + rank)
        ov2 = _perturbed(blk.offd_arrays()[0].copy(), 5 + rank)
        ptr2, col2, val2 = _global_csr(kind, g, p0, world, k=2)
        tp, tc, tv = transposed_csr(n, ptr2, col2, val2)
        fresh = B.DeviceMatrix(B.blocks_from_csr(n, tp, tc, tv, rank=rank, world=world))
        mt.prepare_async("bicgstab")
        x1 = torch.from_numpy(np.random.default_rng(5 + rank).standard_normal(nloc)).cuda()
        ty, tx, tr = (torch.empty(nloc, dtype=torch.float64, device="cuda") for _ in range(3))
        tb = torch.from_numpy(fresh.multiply(np.ones(nloc))).cuda()
        result = torch.zeros(24, dtype=torch.uint8, device="cuda")
        tdv, tov = torch.from_numpy(dv2).cuda(), torch.from_numpy(ov2).cuda()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            dm.set_values_async(tdv, tov if ov2.size else None)
            mt.transpose_values_async(dm)
            mt.multiply_async(x1, ty)
            tx.zero_()
            tr.copy_(tb)
            mt.solve_async("bicgstab", tx, tr, result=result)
        s.synchronize()
        assert _bits(ty) == _bits(fresh.multiply(x1.cpu().numpy())), (kind, rank)
        fx, fr = np.zeros(nloc), tb.cpu().numpy().copy()
        it, _ = fresh.solve("bicgstab", fx, fr)
        assert [B.decode_result(result)["iters"], _bits(tx), _bits(tr)] == [it, _bits(fx), _bits(fr)], (kind, rank)
        # the synchronous refresh back to the first values, with the source gone afterwards
        dm.set_values(blk.diag_arrays()[0].copy(), blk.offd_arrays()[0].copy() if blk.offd.nz else None)
        mt.transpose_values(dm)
        dm.destroy()
        fresh.destroy()
        tp, tc, tv = transposed_csr(n, ptr, col, val)
        fresh = B.DeviceMatrix(B.blocks_from_csr(n, tp, tc, tv, rank=rank, world=world))
        _check(mt, fresh, A, n, nloc, lo, (kind, rank, "refreshed"))
        fresh.destroy()
        mt.destroy()
        if rank == 0:
            print(f"[mgpu {world}] {kind:10s} transpose: bit-identical to the transposed blocks, refresh stream-ordered", flush=True)
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_TRANSPOSE_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
