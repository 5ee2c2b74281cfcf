"""Generate tests/golden/ref_shifted_fixed.npz from the reference's own shifted_lopbicg (shifted_switching_solver.c:20-257), which
oracle/Makefile compiles in place into oracle/_ref/libref_strict.so together with the rest of shifted_switching_solver.c
(BICG_REFERENCE_DIR=<checkout> build()), then
    python tests/golden/make_golden_shifted_fixed.py
Stores, per case, what the REFERENCE produced at P = 1: the return value, the per-iteration sqrt(dot_r/dot_zero) it printed, and
every x_j and the seed residual r (FIXED_CASES) or the SHA-256 of their bytes (FIXED_LARGE_CASES, whose vectors would take
megabytes).  The reference does not report when each shift stopped, so the tests take that from the restatement alone."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
import oracle as O
import shifted_fixed_oracle as OF
from helpers import global_csr
from shifted_fixed_cases import FIXED_CASES, FIXED_LARGE_CASES, GOLDEN_FIXED, fixed_problem


def digest(a):
    return np.str_(hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest())


out = {}
for case in FIXED_CASES + FIXED_LARGE_CASES:
    name = case[0]
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    r = OF.ref_shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=1000)
    out[name + "|ret"] = np.int64(r["ret"])
    out[name + "|res"] = r["res"]
    if case in FIXED_CASES:
        out[name + "|x"] = r["x"]
        out[name + "|r"] = r["r"]
    else:
        out[name + "|x_sha256"] = digest(r["x"])
        out[name + "|r_sha256"] = digest(r["r"])
    print(name, "ret", r["ret"], "printed residuals", len(r["res"]), flush=True)
np.savez_compressed(GOLDEN_FIXED, **out)
print("written", GOLDEN_FIXED, os.path.getsize(GOLDEN_FIXED), "bytes")
