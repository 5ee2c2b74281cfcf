"""Python access to the checker of shifted_lopbicg (shifted_switching_solver.h:11).  TEST INFRASTRUCTURE -- import only from tests/.

  * liboracle_fixed.so   : the C restatement (shifted_fixed_oracle.c), emulating P ranks in one process
  * _ref/libref_strict.so: the reference's own shifted_switching_solver.c compiled in place (oracle/Makefile), P = 1 in-process
liboracle_fixed.so is built by oracle/shifted_fixed.mk (build() runs it); this module builds it itself if it is missing.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import HERE, _csr, _dp, _p, _up, ref_shifted_solve

ORACLE_FIXED_SO = os.path.join(HERE, "liboracle_fixed.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_FIXED_SO):
            subprocess.run(["make", "-C", HERE, "-f", "shifted_fixed.mk", "fixed-oracle"], check=True, capture_output=True)
        L = C.CDLL(ORACLE_FIXED_SO)
        L.orc_shifted_lopbicg.restype = C.c_int
        L.orc_shifted_lopbicg.argtypes = [C.c_int, _dp, _up, _up, C.c_int, _dp, _dp, _dp, C.c_int, C.c_int, C.c_double, C.c_int, _dp,
                                          C.c_int, C.POINTER(C.c_int)]
        _lib = L
    return _lib


def shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, P=1, tol=1e-12, max_iter=1000, x0=None):
    """Restated shifted_lopbicg (shifted_switching_solver.c:20-257) from the initial x_set x0 (None: zero).  Returns dict(ret,
    x (sigma_len x n), r, hist, stop_iter) with ret = iterations performed, hist[k] = dot_r/dot_zero after iteration k and
    stop_iter[j] = the iteration after which shift j stopped (0: never)."""
    ptr, col, val = _csr(ptr, col, val)
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    x = np.zeros((sigma.size, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(sigma.size, n)
    r = np.array(b, dtype=np.float64)
    hist = np.full(max_iter + 2, np.nan)
    stop_iter = (C.c_int * sigma.size)()
    ret = lib().orc_shifted_lopbicg(n, _p(val, _dp), _p(col, _up), _p(ptr, _up), P, _p(x, _dp), _p(r, _dp), _p(sigma, _dp), sigma.size,
                                    seed, tol, max_iter, _p(hist, _dp), hist.size, stop_iter)
    return {"ret": ret, "x": x, "r": r, "hist": hist[:ret + 1], "stop_iter": np.array(stop_iter[:])}


def ref_shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, tol=1e-12, max_iter=1000, x0=None):
    """The reference's own shifted_lopbicg (P = 1) called in-process.  Returns dict(ret, x, r, res) with res = the
    sqrt(dot_r/dot_zero) it printed after every iteration."""
    out = ref_shifted_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=max_iter, variant="shifted_lopbicg", x0=x0)
    return {k: out[k] for k in ("ret", "x", "r", "res")}
