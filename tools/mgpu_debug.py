"""Multi-GPU debug probe: one iteration, compare every vector slice with the oracle."""
import os, sys
import numpy as np, torch, torch.distributed as dist
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mpi_bicgstab_b200 as B, oracle as O
local = int(os.environ.get("LOCAL_RANK", "0")); torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
B.set_options(device=local, quiet=1)
rank, world = B.comm_init_torch()
g = int(sys.argv[1]) if len(sys.argv) > 1 else 14
blk = B.gen_block("stencil15", g, 14.0, rank=rank, world=world)
n, nloc, lo = blk.n, blk.n_loc, int(blk.displs[rank])
g1 = B.gen_block("stencil15", g, 14.0); ptr, col, val = B.block_to_global_csr(g1)
dm = B.DeviceMatrix(blk)
b_ref = O.spmv(n, ptr, col, val, np.ones(n), P=world)
for mega in (0, 1):
    for mi in (1, 2, 3):
        B.set_options(tol=1e-10, max_iter=mi, mega=mega)
        b = dm.spmv(np.ones(nloc)); eb = np.abs(b - b_ref[lo:lo+nloc]).max()
        x = np.zeros(nloc)
        it, st = dm.solve("bicgstab", x, b)
        ref = O.solve("bicgstab", n, ptr, col, val, b_ref, P=world, tol=1e-10, max_iter=mi)
        h = B.last_history()
        ex = np.abs(x - ref["x"][lo:lo+nloc]).max(); er = np.abs(b - ref["r"][lo:lo+nloc]).max()
        bad_x = np.where(np.abs(x - ref["x"][lo:lo+nloc]) > 1e-9)[0]
        print(f"[r{rank}] mega={mega} max_iter={mi}: it={it} hist={np.sqrt(h[1:])} ref={np.sqrt(ref['hist'][1:])} "
              f"err_b={eb:.1e} err_x={ex:.1e} err_r={er:.1e} bad_x_rows={bad_x[:4]}..{bad_x[-2:]} n={bad_x.size}/{nloc}", flush=True)
dm.destroy(); B.comm_finalize(); dist.destroy_process_group()
