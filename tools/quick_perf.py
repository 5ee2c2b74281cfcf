"""Per-iteration time of each loop implementation on one workload (single or multi rank).
usage: quick_perf.py [methods...]   env: QP_KIND/QP_G/QP_P0 (workload), QP_MODES=mega,graph, QP_RESIDENT=1,0, QP_ITERS, BICG_* options"""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B
world = int(os.environ.get("WORLD_SIZE", "1")); rank = int(os.environ.get("RANK", "0")); local = int(os.environ.get("LOCAL_RANK", "0"))
if world > 1:
    import torch, torch.distributed as dist
    os.environ["NCCL_DEBUG"] = "WARN"
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
B.set_options(device=local, quiet=1)
if world > 1:
    B.comm_init_torch()
kind = os.environ.get("QP_KIND", "stencil15"); g = int(os.environ.get("QP_G", "117")); p0 = float(os.environ.get("QP_P0", "14.0"))
if kind == "random":
    g *= world
iters = int(os.environ.get("QP_ITERS", "300"))
modes = os.environ.get("QP_MODES", "mega,graph").split(",")
blk = B.gen_block(kind, g, p0, rank=rank, world=world)
dm = B.DeviceMatrix(blk)
nl = blk.n_loc
resident = [int(v) for v in os.environ.get("QP_RESIDENT", "").split(",") if v != ""]       # e.g. "1,0": persistent kernel with / without resident slices
for method in (sys.argv[1:] or ["bicgstab", "ca_bicgstab", "pipe_bicgstab"]):
    for mode in (modes if not resident else [f"mega/r{r}" for r in resident]):
        kw = dict(mega=1) if mode.startswith("mega") else dict(mega=0)
        if "/r" in mode:
            kw["resident"] = int(mode[-1])
        B.set_options(tol=0.0, max_iter=iters, **kw)
        for rep in range(2):
            b = dm.spmv(np.ones(nl)); x = np.zeros(nl)
            kwargs = dict(krr=50, nrr=3) if method.endswith("rr") else {}
            it, st = dm.solve(method, x, b, **kwargs)
        if rank == 0:
            print(f"[N={world}] {kind} {method:17s} {mode:7s} {st['loop_ms'] / it * 1e3:7.2f} us/it  {it / st['loop_ms'] * 1e3:8.0f} it/s  "
                  f"launches={st['kernel_launches']} res={st['final_res']:.3e}", flush=True)
dm.destroy()
if world > 1:
    B.comm_finalize(); dist.destroy_process_group()
