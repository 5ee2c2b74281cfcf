"""Python access to the checker.  TEST INFRASTRUCTURE -- import only from tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs.  Never from the product.

  * liboracle.so      : the C restatement (bicg_oracle.c), emulating P ranks in one process
  * _ref/libref_*.so  : the reference's own sources compiled in place (oracle/Makefile), P = 1 in-process
  * _ref/ref_driver_* : the same objects behind an in-memory driver + mini-MPI, P >= 1, as a subprocess
"""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liboracle.so")
REF_DIR = os.path.join(HERE, "_ref")

_dp = C.POINTER(C.c_double)
_up = C.POINTER(C.c_uint)


def _p(a, t):
    return a.ctypes.data_as(t)


def have_oracle():
    return os.path.exists(ORACLE_SO)


def have_ref(name="libref_strict.so"):
    return os.path.exists(os.path.join(REF_DIR, name))


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not have_oracle():
            raise RuntimeError(f"{ORACLE_SO} missing: run `make -C oracle oracle`")
        L = C.CDLL(ORACLE_SO)
        common = [C.c_int, _dp, _up, _up, C.c_int, _dp, _dp]
        tail = [C.c_double, C.c_int, _dp, C.c_int]
        for name in ("orc_bicgstab", "orc_ca_bicgstab", "orc_pipe_bicgstab"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = common + tail
        L.orc_pipe_bicgstab_rr.restype = C.c_int
        L.orc_pipe_bicgstab_rr.argtypes = common + [C.c_int, C.c_int] + tail
        L.orc_spmv.restype = None
        L.orc_spmv.argtypes = [C.c_int, _dp, _up, _up, C.c_int, _dp, _dp]
        L.orc_spmv_ld.restype = None
        L.orc_spmv_ld.argtypes = [C.c_int, _dp, _up, _up, _dp, _dp]
        L.orc_ddot.restype = C.c_double
        L.orc_ddot.argtypes = [C.c_int, _dp, _dp]
        L.orc_shifted_lopbicg_switching.restype = C.c_int
        L.orc_shifted_lopbicg_switching.argtypes = [C.c_int, _dp, _up, _up, C.c_int, _dp, _dp, _dp, C.c_int, C.c_int, C.c_double, C.c_int,
                                                    _dp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orc_daxpy.restype = None
        L.orc_daxpy.argtypes = [C.c_int, C.c_double, _dp, _dp]
        L.orc_dscal.restype = None
        L.orc_dscal.argtypes = [C.c_int, C.c_double, _dp]
        L.orc_partition.restype = None
        L.orc_partition.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        _lib = L
    return _lib


def _csr(ptr, col, val):
    return (np.ascontiguousarray(ptr, dtype=np.uint32), np.ascontiguousarray(col, dtype=np.uint32),
            np.ascontiguousarray(val, dtype=np.float64))


def spmv(n, ptr, col, val, x, P=1, long_double=False):
    ptr, col, val = _csr(ptr, col, val)
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.zeros(n)
    if long_double:
        lib().orc_spmv_ld(n, _p(val, _dp), _p(col, _up), _p(ptr, _up), _p(x, _dp), _p(y, _dp))
    else:
        lib().orc_spmv(n, _p(val, _dp), _p(col, _up), _p(ptr, _up), P, _p(x, _dp), _p(y, _dp))
    return y


def solve(method, n, ptr, col, val, b, x0=None, P=1, tol=1e-15, max_iter=1000, krr=0, nrr=0):
    """Run the restated solver.  Returns dict(iters, x, r, hist) with hist[k] = dot_r/dot_zero."""
    ptr, col, val = _csr(ptr, col, val)
    x = np.zeros(n) if x0 is None else np.array(x0, dtype=np.float64)
    r = np.array(b, dtype=np.float64)
    hist = np.full(max_iter + 2, np.nan)
    args = [n, _p(val, _dp), _p(col, _up), _p(ptr, _up), P, _p(x, _dp), _p(r, _dp)]
    tail = [tol, max_iter, _p(hist, _dp), hist.size]
    L = lib()
    if method == "bicgstab":
        it = L.orc_bicgstab(*args, *tail)
    elif method == "ca_bicgstab":
        it = L.orc_ca_bicgstab(*args, *tail)
    elif method == "pipe_bicgstab":
        it = L.orc_pipe_bicgstab(*args, *tail)
    elif method == "pipe_bicgstab_rr":
        it = L.orc_pipe_bicgstab_rr(*args, krr, nrr, *tail)
    else:
        raise ValueError(method)
    return {"iters": it, "x": x, "r": r, "hist": hist[:it + 1]}


# ---- BLAS-1 restatements (vector.c:3-27), in place on contiguous float64 arrays ---------------------------
def _f64(a):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return _p(a, _dp)


def daxpy(a, x, y):
    """y += a * x   (vector.c:3-7)"""
    lib().orc_daxpy(y.size, float(a), _f64(x), _f64(y))


def dscal(a, x):
    """x *= a       (vector.c:17-21)"""
    lib().orc_dscal(x.size, float(a), _f64(x))


def ddot(x, y):
    """sum x_i y_i, left to right (vector.c:9-15)"""
    return float(lib().orc_ddot(x.size, _f64(x), _f64(y)))


def partition(n, P):
    cnt = (C.c_int * P)()
    dsp = (C.c_int * P)()
    lib().orc_partition(n, P, cnt, dsp)
    return np.array(cnt[:]), np.array(dsp[:])


# ---- the compiled reference -------------------------------------------------------------------------------
class _RefCSR(C.Structure):
    _fields_ = [("val", _dp), ("col", _up), ("ptr", _up), ("nz", C.c_uint), ("rows", C.c_uint), ("cols", C.c_uint)]


class _RefInfo(C.Structure):
    _fields_ = [("nz", C.c_uint), ("rows", C.c_uint), ("cols", C.c_uint), ("code", C.c_char * 4),
                ("recvcounts", C.POINTER(C.c_int)), ("displs", C.POINTER(C.c_int))]


_ref_libs = {}


def ref_lib(flavour="strict"):
    if flavour not in _ref_libs:
        path = os.path.join(REF_DIR, f"libref_{flavour}.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} missing: run `make -C oracle ref REF=<checkout of the reference>`")
        L = C.CDLL(path)
        L.orc_ref_config.argtypes = [C.c_double, C.c_int, C.c_int, C.c_int]
        L.orc_ref_hist_res.restype = C.c_double
        L.orc_ref_final_res.restype = C.c_double
        L.orc_ref_avg_time.restype = C.c_double
        L.orc_ref_total_time.restype = C.c_double
        _ref_libs[flavour] = L
    return _ref_libs[flavour]


def ref_solve(method, n, ptr, col, val, b, x0=None, tol=1e-15, max_iter=1000, krr=0, nrr=0, flavour="strict"):
    """The reference's own bicgstab()/... (P = 1) called in-process on an in-memory CSR."""
    L = ref_lib(flavour)
    ptr, col, val = _csr(ptr, col, val)
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
    x = np.zeros(n) if x0 is None else np.array(x0, dtype=np.float64)
    r = np.array(b, dtype=np.float64)
    L.orc_ref_config(tol, max_iter, 1, 1)
    L.orc_ref_hist_reset()
    args = [C.byref(D), C.byref(O), C.byref(info), _p(x, _dp), _p(r, _dp)]
    if method == "pipe_bicgstab_rr":
        it = L.pipe_bicgstab_rr(*args, krr, nrr)
    else:
        it = getattr(L, method)(*args)
    cnt = L.orc_ref_hist_count()
    res = np.array([L.orc_ref_hist_res(i) for i in range(cnt)])
    return {"iters": it, "x": x, "r": r, "res": res, "final_res": L.orc_ref_final_res(),
            "avg_time": L.orc_ref_avg_time(), "total_time": L.orc_ref_total_time()}


def shifted_solve(n, ptr, col, val, b, sigma, seed, P=1, tol=1e-12, max_iter=1000, x0=None):
    """Restated shifted_lopbicg_switching (shifted_switching_solver.c:260-602) from the initial x_set x0 (None: zero).  Returns
    dict(ret, iters, x (sigma_len x n), r, hist, seed, stop_iter)."""
    ptr, col, val = _csr(ptr, col, val)
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    x = np.zeros((sigma.size, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(sigma.size, n)
    r = np.array(b, dtype=np.float64)
    hist = np.full(max_iter + 2, np.nan)
    seed_out = C.c_int(seed)
    stop_iter = (C.c_int * sigma.size)()
    ret = lib().orc_shifted_lopbicg_switching(n, _p(val, _dp), _p(col, _up), _p(ptr, _up), P, _p(x, _dp), _p(r, _dp), _p(sigma, _dp),
                                              sigma.size, seed, tol, max_iter, _p(hist, _dp), hist.size, C.byref(seed_out), stop_iter)
    return {"ret": ret, "iters": ret - 1, "x": x, "r": r, "hist": hist[:ret], "seed": seed_out.value, "stop_iter": np.array(stop_iter[:])}


def ref_shifted_solve(n, ptr, col, val, b, sigma, seed, tol=1e-12, max_iter=1000, flavour="strict", variant="shifted_lopbicg_switching",
                      x0=None):
    """The reference's own shifted_lopbicg_switching() (or its _noovlp twin, shifted_switching_solver.c:611) at P = 1, called
    in-process on an in-memory CSR, from the initial x_set x0 (None: zero)."""
    L = ref_lib(flavour)
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
    fn = getattr(L, variant)
    fn.restype = C.c_int
    ret = fn(C.byref(D), C.byref(O), C.byref(info), _p(x, _dp), _p(r, _dp), _p(sigma, _dp), int(sigma.size), int(seed))
    cnt = L.orc_ref_hist_count()
    res = np.array([L.orc_ref_hist_res(i) for i in range(cnt)])
    return {"ret": ret, "iters": ret - 1, "x": x, "r": r, "res": res}


def write_csr_bin(path, n, ptr, col, val):
    ptr, col, val = _csr(ptr, col, val)
    with open(path, "wb") as f:
        np.array([n, int(ptr[-1])], dtype=np.int64).tofile(f)
        ptr.tofile(f)
        col.tofile(f)
        if (n + 1 + int(ptr[-1])) % 2:
            np.zeros(1, dtype=np.uint32).tofile(f)
        val.tofile(f)


def ref_driver(method, csr_bin, P=1, rhs="a1", tol=1e-15, max_iter=1000, krr=0, nrr=0, flavour="strict",
               want_vectors=True, pin=False, timeout=3600):
    """Run the compiled reference with P ranks (fork + shm mini-MPI) on a binary CSR file."""
    exe = os.path.join(REF_DIR, f"ref_driver_{flavour}")
    if not os.path.exists(exe):
        raise RuntimeError(f"{exe} missing")
    env = dict(os.environ, MINI_MPI_NP=str(P), REF_EPS=repr(tol), REF_MAX_ITER=str(max_iter), REF_OUT_ITER="1",
               REF_QUIET="1", MALLOC_MMAP_THRESHOLD_="0", MINI_MPI_PIN="1" if pin else "0")
    with tempfile.TemporaryDirectory() as td:
        prefix = os.path.join(td, "out") if want_vectors else "-"
        cmd = [exe, csr_bin, method, rhs, prefix]
        if method == "pipe_bicgstab_rr":
            cmd += [str(krr), str(nrr)]
        out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=timeout, check=True)
        line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
        res = json.loads(line)
        if want_vectors:
            raw = np.fromfile(prefix + ".hist", dtype=np.uint8)
            cnt = int(np.frombuffer(raw[:4].tobytes(), dtype=np.int32)[0])
            rec = np.frombuffer(raw[4:4 + 12 * cnt].tobytes(), dtype=np.dtype([("k", "<i4"), ("res", "<f8")]))
            res["res"] = rec["res"].copy()
            res["x"] = np.concatenate([np.fromfile(f"{prefix}.x.{p}") for p in range(P)])
            res["r"] = np.concatenate([np.fromfile(f"{prefix}.r.{p}") for p in range(P)])
    return res
