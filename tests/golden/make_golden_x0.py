"""Generate tests/golden/ref_x0.npz from the reference's own solvers, compiled in place by build() from a checkout of the
reference (BICG_REFERENCE_DIR=<checkout>), run from nonzero initial guesses:
    python tests/golden/make_golden_x0.py
Stores, per problem of helpers.X0_PLAIN / X0_SHIFTED, the initial guess and what the REFERENCE produced from it at P = 1: the
iteration count (plain solvers) or return value (shifted), x, r and the per-iteration sqrt(dot_r/dot_zero) it printed.  Plain
solvers: bicgstab, ca_bicgstab, pipe_bicgstab and pipe_bicgstab_rr from a standard-normal x0 and from a warm start.  Shifted
solvers: shifted_lopbicg_switching, shifted_lopbicg, shifted_lopbicgstab and shifted_pipe_lopbicgstab from 0.1 standard normal."""
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
import shifted_lop_oracle as OL
from helpers import (METHODS, X0_GOLDEN, X0_KINDS, X0_PLAIN, X0_PLAIN_MAX_ITER, X0_PLAIN_TOL, X0_RR, X0_SHIFTED, X0_SHIFTED_MAX_ITER,
                     X0_SHIFTED_TOL, global_csr, initial_guess, initial_x_set, shifted_problem)

out = {}
kind, g, p0, gseed = X0_PLAIN
_, n, ptr, col, val = global_csr(B, kind, g, p0, seed=gseed)
b = O.spmv(n, ptr, col, val, np.ones(n))
for x0_kind in X0_KINDS:
    x0 = initial_guess(x0_kind, n)
    out[f"plain|{x0_kind}|x0"] = x0
    for method in METHODS:
        kw = X0_RR if method == "pipe_bicgstab_rr" else {}
        r = O.ref_solve(method, n, ptr, col, val, b, x0=x0, tol=X0_PLAIN_TOL, max_iter=X0_PLAIN_MAX_ITER, **kw)
        key = f"plain|{x0_kind}|{method}"
        out[key + "|iters"] = np.int64(r["iters"])
        out[key + "|res"], out[key + "|x"], out[key + "|r"] = r["res"], r["x"], r["r"]
        print(key, r["iters"], len(r["res"]), flush=True)

kind, g, p0, L, scale, seed = X0_SHIFTED
_, n, ptr, col, val = global_csr(B, kind, g, p0)
sigma, b = shifted_problem(O, n, ptr, col, val, L, scale, seed)
x0 = initial_x_set(L, n)
out["shifted|x0"] = x0
args, kw = (n, ptr, col, val, b, sigma, seed), dict(tol=X0_SHIFTED_TOL, max_iter=X0_SHIFTED_MAX_ITER, x0=x0)
for method, r in (("shifted_lopbicg_switching", O.ref_shifted_solve(*args, **kw)),
                  ("shifted_lopbicg", OF.ref_shifted_fixed_solve(*args, **kw)),
                  ("shifted_lopbicgstab", OL.ref_shifted_lop_solve(*args, "shifted_lopbicgstab", **kw)),
                  ("shifted_pipe_lopbicgstab", OL.ref_shifted_lop_solve(*args, "shifted_pipe_lopbicgstab", **kw))):
    key = f"shifted|{method}"
    out[key + "|ret"] = np.int64(r["ret"])
    out[key + "|res"], out[key + "|x"], out[key + "|r"] = r["res"], r["x"], r["r"]
    print(key, r["ret"], len(r["res"]), flush=True)
np.savez_compressed(X0_GOLDEN, **out)
print("written", X0_GOLDEN, os.path.getsize(X0_GOLDEN), "bytes")
