"""Multi-GPU worker of the asynchronous solve (one process per GPU, torchrun + NCCL for the bootstrap only): on its row block every
rank runs each method synchronously (bicg_solve with device vectors) and asynchronously on torch's current stream
(bicg_solve_async), on the persistent kernel and on the kernel-per-phase path (WHILE node), and requires x, r, the history and the
result record to be bit-identical; then it captures {r <- b_buf; x <- 0; solve_async} into a torch CUDA graph and replays it with
three different b, each equal to the synchronous solve of that b.  A stencil and random n = 3001 (odd n_loc on some rank)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from helpers import METHODS

RR = dict(krr=10, nrr=3)
PROBLEMS = [("stencil15", 12, 14.0), ("random", 3001, 8)]
PATHS = {"persistent": dict(mega=1), "graph": dict(mega=0)}


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _sync(dm, method, b):
    x, r = torch.zeros_like(b), b.clone()
    it, st = dm.solve(method, x, r, **(RR if method.endswith("rr") else {}))
    return dict(x=_bits(x.cpu()), r=_bits(r.cpu()), hist=_bits(B.last_history()), iters=it, conv=st["converged"],
                res=_bits(st["final_res"]))


def _record(x, r, dm, res):
    d = B.decode_result(res)
    assert d["error"] == 0, d
    return dict(x=_bits(x.cpu()), r=_bits(r.cpu()), hist=_bits(dm.history()), iters=d["iters"], conv=d["converged"],
                res=_bits(d["final_res"]))


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1, tol=1e-10, max_iter=1000)
    rank, world = B.comm_init_torch()
    for kind, g, p0 in PROBLEMS:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
        b = torch.from_numpy(ref_dm.spmv(np.ones(blk.n_loc))).cuda()
        bs = [b, b * 0.5 + 1.0, b - 0.25]
        for path, opts in PATHS.items():
            B.set_options(**opts)
            for method in METHODS:
                kw = RR if method.endswith("rr") else {}
                want = [_sync(ref_dm, method, bb) for bb in bs]
                x, r = torch.zeros_like(b), b.clone()
                res = dm.solve_async(method, x, r, **kw)
                torch.cuda.synchronize()
                assert _record(x, r, dm, res) == want[0], (kind, path, method, rank, "async")
                dm.prepare_async(method)
                b_buf, x, r = torch.zeros_like(b), torch.zeros_like(b), torch.zeros_like(b)
                res = torch.zeros(24, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    r.copy_(b_buf)
                    x.zero_()
                    dm.solve_async(method, x, r, result=res, **kw)
                for i, bb in enumerate(bs):
                    b_buf.copy_(bb)
                    graph.replay()
                    torch.cuda.synchronize()
                    assert _record(x, r, dm, res) == want[i], (kind, path, method, rank, "replay", i)
                del graph
                if rank == 0:
                    print(f"[mgpu {world}] {kind} {path} {method}: async and 3 replays = sync ({want[0]['iters']})", flush=True)
        B.set_options(mega=1)
        ref_dm.destroy(); dm.destroy()
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_ASYNC_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
