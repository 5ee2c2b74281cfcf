"""Throughput of the shifted solvers on the T' matrix (1 GPU): iterations/s and effective GB/s on each method's algorithmic bytes
per iteration (DESIGN.md section 3.4 / 3.5):
    switching  24 nnz + 32 n (active shifts) + 200 n (seed BiCGStab: two SpMVs + its vector phases)
    fixed      the same (shifted_lopbicg runs the switching solver's kernels without the seed switch)
    lop        24 nnz + 32 n (L - 1) + 168 n
    pipe_lop   24 nnz + 32 n (L - 1) + 240 n
usage: shifted_perf.py [--method switching|fixed|lop|pipe_lop] [L ...]   env: SP_G (grid size, default 117)"""
import argparse, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B
METHODS = {"switching": "shifted_lopbicg_switching", "fixed": "shifted_lopbicg", "lop": "shifted_lopbicgstab",
           "pipe_lop": "shifted_pipe_lopbicgstab"}
ap = argparse.ArgumentParser()
ap.add_argument("--method", choices=sorted(METHODS), default="switching")
ap.add_argument("L", nargs="*", type=int, default=[16, 64])
args = ap.parse_args()
g = int(os.environ.get("SP_G", "117"))
B.set_options(quiet=1)
blk = B.gen_block("stencil15", g, 14.0)
n, nnz = blk.n, blk.nnz_loc
dm = B.DeviceMatrix(blk)
ones = np.ones(n)
for L in args.L:
    sigma = (np.arange(L) + 1) * (0.01 / L)                   # main_shifted.c:95-99
    b = dm.spmv(ones) + sigma[0] * ones
    B.set_options(shift_tol=1e-8, shift_max_iter=300)
    for rep in range(2):
        x = np.zeros((L, n)); r = b.copy()
        k, st = dm.shifted_solve(METHODS[args.method], x, r, sigma, 0)
    if args.method in ("switching", "fixed"):
        it = k - 1 if args.method == "switching" else k
        seed, stop = B.last_shift_info(L)
        active = sum(min(int(s) if s else it, it) for j, s in enumerate(stop) if j != 0) / max(it, 1)      # average active shifts per iteration
        bytes_it = 24.0 * nnz + 32.0 * n * active + 200.0 * n
        extra = f"avg active shifts {active:.1f}, final seed {seed}"
    else:
        it = k
        bytes_it = 24.0 * nnz + 32.0 * n * (L - 1) + (168.0 if args.method == "lop" else 240.0) * n
        extra = f"{L - 1} shifts"
    us = st["loop_ms"] * 1e3 / max(it, 1)
    print(f"[shifted {args.method}] T' g={g} n={n} L={L}: {it} iterations, {us:.1f} us/iteration, {1e6 / us:.0f} it/s, {extra}, "
          f"{bytes_it / us / 1e3:.0f} GB/s on algorithmic bytes ({bytes_it / 1e6:.0f} MB/iteration), launches {st['kernel_launches']}, "
          f"res {st['final_res']:.2e}", flush=True)
dm.destroy()
