"""Multi-GPU worker of the asynchronous shifted solve (one process per GPU, torchrun + NCCL for the bootstrap only): on its row
block every rank runs each shifted method synchronously (bicg_shifted_solve_dev) and asynchronously on torch's current stream
(bicg_shifted_solve_async), from a nonzero x_set, and requires x_set, r, stop_iter, the history and the result record to be
bit-identical; then it captures {r <- b_buf; x_set <- x0; shifted_solve_async} into a torch CUDA graph and replays it with three
different b and sigma, each equal to the synchronous solve of those inputs.  A stencil and random n = 3001 (odd n_loc on some
rank)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B

METHODS = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]
PROBLEMS = [("stencil15", 12, 14.0, 5, 0.01 / 5, 0), ("random", 3001, 8, 6, 0.01, 5)]


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _sync(dm, method, x0, b, sigma, seed):
    x, r = x0.clone(), b.clone()
    k, st = dm.shifted_solve(method, x, r, sigma.cpu().numpy(), seed)
    s, stop = B.last_shift_info(sigma.numel())
    return dict(x=_bits(x), r=_bits(r), hist=_bits(B.last_history()), stop=list(stop), ret=k, iters=st["iters"],
                conv=st["converged"], seed=s, res=_bits(st["final_res"]))


def _record(dm, x, r, res, stop):
    d = B.decode_shift_result(res)
    assert d["error"] == 0, d
    return dict(x=_bits(x), r=_bits(r), hist=_bits(dm.shift_history()), stop=[int(v) for v in stop.cpu()], ret=d["ret"],
                iters=d["iters"], conv=d["converged"], seed=d["seed"], res=_bits(d["final_res"]))


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B.set_options(device=local, quiet=1, shift_tol=1e-12, shift_max_iter=1000)
    rank, world = B.comm_init_torch()
    for kind, g, p0, L, scale, seed in PROBLEMS:
        blk = B.gen_block(kind, g, p0, rank=rank, world=world)
        ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
        n = blk.n_loc
        b = torch.from_numpy(ref_dm.spmv(np.ones(n))).cuda()
        sigma = torch.from_numpy((np.arange(L) + 1) * scale).cuda()
        x0 = 0.1 * torch.from_numpy(np.random.default_rng(n + L).standard_normal((L, n))).cuda()
        inputs = [(b + sigma[seed], sigma), (b * 0.5 + 1.0, sigma * 0.75), (b - 0.25, sigma + 0.05)]
        for method in METHODS:
            want = [_sync(ref_dm, method, x0, bb, sg, seed) for bb, sg in inputs]
            x, r = x0.clone(), inputs[0][0].clone()
            stop = torch.zeros(L, dtype=torch.int32, device="cuda")
            res = dm.shifted_solve_async(method, x, r, inputs[0][1].clone(), seed, stop_iter=stop)
            torch.cuda.synchronize()
            assert _record(dm, x, r, res, stop) == want[0], (kind, method, rank, "async")
            dm.prepare_shifted_async(method, L)
            b_buf, s_buf = torch.zeros_like(b), torch.zeros_like(sigma)
            x, r = torch.zeros_like(x0), torch.zeros_like(b)
            res = torch.zeros(32, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                r.copy_(b_buf)
                x.copy_(x0)
                dm.shifted_solve_async(method, x, r, s_buf, seed, result=res, stop_iter=stop)
            for i, (bb, sg) in enumerate(inputs):
                b_buf.copy_(bb); s_buf.copy_(sg)
                graph.replay()
                torch.cuda.synchronize()
                assert _record(dm, x, r, res, stop) == want[i], (kind, method, rank, "replay", i)
            del graph
            if rank == 0:
                print(f"[mgpu {world}] {kind} {method}: async and 3 replays = sync ({want[0]['ret']})", flush=True)
        ref_dm.destroy(); dm.destroy()
    B.comm_finalize()
    dist.barrier()
    if rank == 0:
        print("MGPU_SHIFTED_ASYNC_OK", world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
