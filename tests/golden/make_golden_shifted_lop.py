"""Generate tests/golden/ref_shifted_lop_<function>.npz (and test_shifted_convdiff16.mtx) from the reference's own shifted_solver.c
(shifted_lopbicgstab and its twins, compiled in place into oracle/_ref/libref_lop_strict.so, and the unchanged test_shifted.c on
the mini-MPI, oracle/_ref/ref_test_shifted_stock, both built by oracle/shifted_lop.mk; BICG_REFERENCE_DIR=<checkout> build()), then
    python tests/golden/make_golden_shifted_lop.py
Stores, per case and for all five reference functions, what the REFERENCE produced: return value, every x_j, the seed residual
r and the per-iteration sqrt(dot_r/dot_zero) history; and the `Total iter` the unchanged test_shifted.c prints on the .mtx file."""
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
import oracle as O
import shifted_lop_oracle as OL
from helpers import global_csr
from shifted_lop_cases import SHIFTED_LOP_CASES, SHIFTED_LOP_MTX, SHIFTED_LOP_VARIANTS, golden_path, mtx_path, shifted_lop_problem

out = {v: {} for v in SHIFTED_LOP_VARIANTS}
for case in SHIFTED_LOP_CASES:
    name = case[0]
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    for variant in SHIFTED_LOP_VARIANTS:
        r = OL.ref_shifted_lop_solve(n, ptr, col, val, b, sigma, seed, variant, tol=1e-12, max_iter=1000)
        out[variant][name + "|ret"] = np.int64(r["ret"])
        out[variant][name + "|x"] = r["x"]
        out[variant][name + "|r"] = r["r"]
        out[variant][name + "|res"] = r["res"]
        print(name, variant, r["ret"], len(r["res"]))

# test_shifted.c's own set-up (SIGMA_LENGTH 5, sigma_i = 0.01 i + 0.01, seed 0, x = 1) on a small Matrix-Market file
kind, g, p0 = SHIFTED_LOP_MTX
blk, n, ptr, col, val = global_csr(B, kind, g, p0)
mtx = mtx_path()
with open(mtx, "w") as f:
    f.write("%%MatrixMarket matrix coordinate real general\n")
    f.write(f"{n} {n} {int(ptr[-1])}\n")
    for i in range(n):
        for k in range(int(ptr[i]), int(ptr[i + 1])):
            f.write(f"{i + 1} {int(col[k]) + 1} {float(val[k])!r}\n")
env = dict(os.environ, MINI_MPI_NP="1")
p = subprocess.run([os.path.join(ROOT, "oracle", "_ref", "ref_test_shifted_stock"), mtx], capture_output=True, text=True, env=env,
                   check=True)
total_iter = int(re.search(r"Total iter\s*:\s*(\d+)", p.stdout).group(1))
out["shifted_pipe_lopbicgstab_nooverlap"]["test_shifted_mtx|total_iter"] = np.int64(total_iter)      # what test_shifted.c:127 calls
print("test_shifted.c on", os.path.basename(mtx), ":", total_iter, "iterations")
for variant, arrays in out.items():
    np.savez_compressed(golden_path(variant), **arrays)
    print("written", golden_path(variant), len(arrays), "arrays")
