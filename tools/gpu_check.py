"""Development probe run on the GPU box: autotune table + SpMV / solve timings on the BASELINE shapes."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B

PEAK = 6569.3
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass

which = sys.argv[1:] or ["transport", "laplace"]
B.set_options(quiet=1, verbose=1)
for w in which:
    t0 = time.time()
    if w == "transport":
        blk = B.gen_block("stencil15", 117, 14.0)
    elif w == "laplace":
        blk = B.gen_block("laplace5", 2000)
    elif w == "random":
        blk = B.gen_block("random", 2_000_000, 32)
    print(f"== {w}: n={blk.n} nnz={blk.nnz_loc} gen {time.time() - t0:.1f}s", flush=True)
    dm = B.DeviceMatrix(blk)
    ms, by = dm.spmv_time(50)
    print(f"spmv+dot: {ms * 1e3:.1f} us, {by / ms / 1e6:.0f} GB/s algorithmic = {by / ms / 1e6 / PEAK:.3f} of measured HBM peak", flush=True)
    n = blk.n
    for method in ("bicgstab", "ca_bicgstab", "pipe_bicgstab"):
        for mega in (1, 0):
            B.set_options(tol=0.0, max_iter=200, mega=mega)
            b = dm.spmv(np.ones(n))
            x = np.zeros(n)
            it, st = dm.solve(method, x, b)
            it, st = dm.solve(method, np.zeros(n), dm.spmv(np.ones(n)))
            per = st["loop_ms"] / max(it, 1) * 1e3
            nb = {"bicgstab": 160, "ca_bicgstab": 216, "pipe_bicgstab": 232}[method]
            byt = 24 * blk.nnz_loc + nb * n
            print(f"{method:14s} mode={['graph', 'mega'][mega]}: {it} it, {per:.1f} us/it, {1e6 / per:.0f} it/s, "
                  f"{byt / per / 1e3:.0f} GB/s = {byt / per / 1e3 / PEAK:.3f} of peak, launches {st['kernel_launches']}", flush=True)
    B.set_options(mega=1)
    ms3, cnt3 = dm.profile("bicgstab", 100)
    print("profile bicgstab 100 it: class ms", [round(v, 3) for v in ms3], "launches", cnt3,
          "avg us", [round(1e3 * a / max(b_, 1), 1) for a, b_ in zip(ms3, cnt3)], flush=True)
    dm.destroy()
    blk.free()
