"""Python access to the checker of the LOP family of shifted_solver.h.  TEST INFRASTRUCTURE -- import only from tests/.

  * liboracle_lop.so         : the C restatement (shifted_lop_oracle.c), emulating P ranks in one process
  * _ref/libref_lop_strict.so: the reference's own shifted_solver.c compiled in place, P = 1 in-process
Both are built by oracle/shifted_lop.mk (build() runs it); this module builds the restatement itself if it is missing.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import HERE, REF_DIR, _RefCSR, _RefInfo, _csr, _dp, _p, _up

ORACLE_LOP_SO = os.path.join(HERE, "liboracle_lop.so")
VARIANTS = ("shifted_lopbicgstab", "shifted_lopbicgstab_v2", "shifted_lopbicgstab_nooverlap", "shifted_pipe_lopbicgstab",
            "shifted_pipe_lopbicgstab_nooverlap")

_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_LOP_SO):
            subprocess.run(["make", "-C", HERE, "-f", "shifted_lop.mk", "lop-oracle"], check=True, capture_output=True)
        L = C.CDLL(ORACLE_LOP_SO)
        for name in ("orc_shifted_lopbicgstab", "orc_shifted_pipe_lopbicgstab"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [C.c_int, _dp, _up, _up, C.c_int, _dp, _dp, _dp, C.c_int, C.c_int, C.c_double, C.c_int, _dp,
                                         C.c_int]
        _lib = L
    return _lib


def shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=False, P=1, tol=1e-12, max_iter=1000, x0=None):
    """Restated shifted_lopbicgstab (shifted_solver.c:182-354) or, with pipe, shifted_pipe_lopbicgstab (:703-895), from the
    initial x_set x0 (None: zero).  Returns
    dict(ret, x (sigma_len x n), r, hist) with ret = iterations performed and hist[k] = dot_r/dot_zero."""
    ptr, col, val = _csr(ptr, col, val)
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    x = np.zeros((sigma.size, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(sigma.size, n)
    r = np.array(b, dtype=np.float64)
    hist = np.full(max_iter + 2, np.nan)
    fn = lib().orc_shifted_pipe_lopbicgstab if pipe else lib().orc_shifted_lopbicgstab
    ret = fn(n, _p(val, _dp), _p(col, _up), _p(ptr, _up), P, _p(x, _dp), _p(r, _dp), _p(sigma, _dp), sigma.size, seed, tol, max_iter,
             _p(hist, _dp), hist.size)
    return {"ret": ret, "x": x, "r": r, "hist": hist[:ret + 1]}


def have_ref():
    return os.path.exists(os.path.join(REF_DIR, "libref_lop_strict.so"))


def ref_lib():
    global _ref
    if _ref is None:
        path = os.path.join(REF_DIR, "libref_lop_strict.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} missing: run `make -C oracle -f shifted_lop.mk lop-ref REF=<checkout of the reference>`")
        L = C.CDLL(path)
        L.orc_ref_config.argtypes = [C.c_double, C.c_int, C.c_int, C.c_int]
        L.orc_ref_hist_res.restype = C.c_double
        for v in VARIANTS:
            getattr(L, v).restype = C.c_int
        _ref = L
    return _ref


def ref_shifted_lop_solve(n, ptr, col, val, b, sigma, seed, variant, tol=1e-12, max_iter=1000, x0=None):
    """The reference's own shifted_solver.h function `variant` (P = 1) called in-process on an in-memory CSR, from the initial
    x_set x0 (None: zero).  Returns
    dict(ret, x (sigma_len x n), r, res) with res = the sqrt(dot_r/dot_zero) it printed after every iteration."""
    L = ref_lib()
    ptr, col, val = _csr(ptr, col, val)
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    D, O, info = _RefCSR(), _RefCSR(), _RefInfo()
    D.val, D.col, D.ptr = _p(val, _dp), _p(col, _up), _p(ptr, _up)
    D.nz, D.rows, D.cols = int(ptr[-1]), n, n
    zero_ptr = np.zeros(n + 1, dtype=np.uint32)
    one_d, one_u = np.zeros(1), np.zeros(1, dtype=np.uint32)
    O.val, O.col, O.ptr = _p(one_d, _dp), _p(one_u, _up), _p(zero_ptr, _up)
    O.nz, O.rows, O.cols = 0, n, n
    rc = (C.c_int * 1)(n)
    ds = (C.c_int * 1)(0)
    info.nz, info.rows, info.cols, info.code = int(ptr[-1]), n, n, b"MCRG"
    info.recvcounts, info.displs = C.cast(rc, C.POINTER(C.c_int)), C.cast(ds, C.POINTER(C.c_int))
    x = np.zeros((sigma.size, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(sigma.size, n)
    r = np.array(b, dtype=np.float64)
    L.orc_ref_config(tol, max_iter, 1, 1)
    L.orc_ref_hist_reset()
    ret = getattr(L, variant)(C.byref(D), C.byref(O), C.byref(info), _p(x, _dp), _p(r, _dp), _p(sigma, _dp), int(sigma.size), int(seed))
    res = np.array([L.orc_ref_hist_res(i) for i in range(L.orc_ref_hist_count())])
    return {"ret": ret, "x": x, "r": r, "res": res}
