"""Short, deterministic run for ncu: one matrix, a few iterations of one method.
usage: prof_run.py <workload> <method> <iters> <mode: mega|graph>"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B

workload = sys.argv[1] if len(sys.argv) > 1 else "transport"
method = sys.argv[2] if len(sys.argv) > 2 else "bicgstab"
iters = int(sys.argv[3]) if len(sys.argv) > 3 else 30
mode = sys.argv[4] if len(sys.argv) > 4 else "graph"
B.set_options(quiet=1, tol=0.0, max_iter=iters, mega=1 if mode == "mega" else 0)
blk = {"transport": lambda: B.gen_block("stencil15", 117, 14.0), "laplace": lambda: B.gen_block("laplace5", 2000),
       "random": lambda: B.gen_block("random", 2_000_000, 32)}[workload]()
dm = B.DeviceMatrix(blk)
b = dm.spmv(np.ones(blk.n))
x = np.zeros(blk.n)
it, st = dm.solve(method, x, b)
print(workload, method, mode, it, st["loop_ms"] / it * 1e3, "us/it", "lanes", st["spmv_lanes"], "launches", st["kernel_launches"])
