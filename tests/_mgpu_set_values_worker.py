"""Multi-GPU worker for value updates on a resident matrix (one process per GPU, torchrun + NCCL for the bootstrap only).  Every
rank sets new diag and offd values of its own rows (host arrays on one matrix, CUDA tensors on the other), then runs a
persistent-kernel solve, a kernel-per-phase solve and a shifted solve, and shifts its diagonal: every result must be bit-identical
to a handle freshly created from blocks holding the same values, on every rank."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from helpers import RR, initial_guess, initial_x_set


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _perturbed(v, k):
    return v * (1.0 + ((np.arange(v.size) * (2 * k + 1) + k) % 7) / 64.0)


def _with_values(blk, dv, ov):
    blk.diag_arrays()[0][:] = dv
    if ov.size:
        blk.offd_arrays()[0][:] = ov
    return blk


def _results(dm, nloc):
    """persistent-kernel bicgstab, kernel-per-phase pipe_bicgstab_rr, shifted_lopbicgstab: everything they return, as bytes."""
    out = []
    b = dm.spmv(np.ones(nloc))
    out.append(_bits(b))
    x0 = initial_guess("warm", nloc, seed=B.lib.bicg_comm_rank())
    for mega, method in ((1, "bicgstab"), (0, "pipe_bicgstab_rr")):
        B.set_options(mega=mega)
        x, r = x0.copy(), b.copy()
        it, st = dm.solve(method, x, r, **(RR if method.endswith("rr") else {}))
        out += [it, st["kernel_launches"] <= 8, _bits(x), _bits(r), _bits(B.last_history())]
    B.set_options(mega=1)
    sigma = np.array([0.0, 0.25, 1.0])
    xs = initial_x_set(sigma.size, nloc)
    k, _ = dm.shifted_solve("shifted_lopbicgstab", xs, b.copy(), sigma, 0)
    out += [k, _bits(xs), _bits(B.last_history())]
    return out


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1)
    rank, world = B.comm_init_torch()
    B.set_options(tol=1e-10, max_iter=600, mega=1, resident=0, cache=1)
    for kind, g, p0, src in [("stencil15", 40, 14.0, "numpy"), ("convdiff", 200, 1.5, "torch")]:
        make = lambda: B.gen_block(kind, g, p0, rank=rank, world=world)
        blk = make()
        dv, ov = blk.diag_arrays()[0].copy(), blk.offd_arrays()[0].copy()
        assert ov.size > 0, (kind, rank)
        dv2, ov2 = _perturbed(dv, 2 + rank), _perturbed(ov, 5 + rank)
        dm = B.DeviceMatrix(blk)
        fresh = B.DeviceMatrix(_with_values(make(), dv2, ov2))
        before = _results(dm, blk.n_loc)
        if src == "torch":
            dm.set_values(torch.from_numpy(dv2).cuda(), torch.from_numpy(ov2).cuda())
        else:
            dm.set_values(dv2, ov2)
        got, want = _results(dm, blk.n_loc), _results(fresh, blk.n_loc)
        assert got == want, (kind, rank)
        assert got != before, (kind, rank)
        assert got[2] and not got[7], (kind, rank, "loop paths")
        fresh.destroy()
        # each rank shifts the diagonal of its own rows
        ref = _with_values(make(), dv2, ov2)
        for sigma in (0.5, -0.25):
            dm.shift_diagonal(sigma)
            B.lib.csr_shift_diagonal(C.byref(ref.diag), sigma)
            fresh = B.DeviceMatrix(ref)
            assert _results(dm, blk.n_loc) == _results(fresh, blk.n_loc), (kind, rank, sigma)
            fresh.destroy()
        dm.destroy()
        if rank == 0:
            print(f"[mgpu {world}] {kind:10s} set_values ({src}) and shift_diagonal: bit-identical to fresh handles", flush=True)
    B.set_options(resident=1)
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SET_VALUES_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
