"""CPU: the batched multiply in the C ABI -- bicg_matrix_multiply and _async are declared, exported and bound, a null handle / x /
y, nvec <= 0 or overlapping x and y return -1 before the device is touched, a valid call without a GPU exits 1, and the Python
wrappers (DeviceMatrix.multiply / multiply_async) reject bad arrays before they call the library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTOS = ("int bicg_matrix_multiply(bicg_matrix *m, int nvec, const double *x, double *y, double alpha, double beta, "
          "const double *sigma, int device_vectors);",
          "int bicg_matrix_multiply_async(bicg_matrix *m, int nvec, const double *x, double *y, double alpha, double beta, "
          "const double *sigma, void *stream);")
NAMES = ("bicg_matrix_multiply", "bicg_matrix_multiply_async")


def test_declared_exported_and_bound(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    exported = _exported(B)
    for proto, name in zip(PROTOS, NAMES):
        assert " ".join(proto.split()) in header, proto
        assert name in exported and name in B.SYMBOLS, name


def _handle(n_loc):
    """A zeroed stand-in for a handle, never used past the argument checks, with n_loc (the struct's third int) set."""
    h = C.create_string_buffer(4096)
    C.c_int.from_buffer(h, 8).value = n_loc
    return h, C.addressof(h)


def test_bad_arguments_without_gpu(B):
    """Every -1 case returns before the device is touched, in both calls (the synchronous one for host and device vectors)."""
    h, hp = _handle(4)
    buf = (C.c_double * 64)()
    base = C.addressof(buf)
    x, y = base, base + 8 * 32                     # 2 x 4 doubles each, far apart
    sig = (C.c_double * 8)()
    calls = [lambda *a: B.lib.bicg_matrix_multiply(*a, 0), lambda *a: B.lib.bicg_matrix_multiply(*a, 1),
             lambda *a: B.lib.bicg_matrix_multiply_async(*a, None)]
    for call in calls:
        for args in ((None, 2, x, y), (hp, 2, None, y), (hp, 2, x, None),           # null handle / x / y
                     (hp, 0, x, y), (hp, -3, x, y),                                 # nvec <= 0
                     (hp, 2, x, x), (hp, 2, x, x + 8 * 7), (hp, 2, x + 8 * 7, x),   # x and y overlap
                     (hp, 1, x, x + 8 * 3)):
            for s in (None, sig):
                assert call(args[0], args[1], args[2], args[3], 1.0, 0.0, s) == -1, args


@pytest.mark.parametrize("call", ["B.lib.bicg_matrix_multiply(hp, 2, x, y, 1.0, 0.0, None, 0)",
                                  "B.lib.bicg_matrix_multiply(hp, 2, x, y, -1.0, 1.0, s, 1)",
                                  "B.lib.bicg_matrix_multiply_async(hp, 2, x, y, 1.0, 0.0, None, None)"])
def test_valid_call_fails_loudly_without_gpu(B, call):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys, ctypes as C; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; "
            "h = C.create_string_buffer(4096); C.c_int.from_buffer(h, 8).value = 4; hp = C.addressof(h); "
            "b = (C.c_double * 64)(); x = C.addressof(b); y = x + 8 * 32; s = (C.c_double * 2)(); "
            "%s; print('RETURNED')" % (ROOT, call))
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


# ---- the Python wrappers reject bad vectors before the library sees them ---------------------------------------------------
N = 64


@pytest.fixture
def dm(B):
    """A DeviceMatrix of a one-rank block whose handle is never used."""
    import scipy.sparse as sp
    A = sp.diags([-np.ones(N - 1), 4.0 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1], format="csr")
    blk = B.blocks_from_csr(N, A.indptr, A.indices, A.data)
    d = B.DeviceMatrix.__new__(B.DeviceMatrix)
    d.blk, d.h = blk, None
    yield d
    d.h = None


def _reject(fn, exc, text):
    with pytest.raises(exc, match=text):
        fn()


def test_multiply_rejects_bad_arrays(B, dm):
    import torch
    f = dm.multiply
    x, y = np.ones((3, N)), np.zeros((3, N))
    _reject(lambda: f(x.astype(np.float32)), TypeError, "float64")                         # wrong dtype
    _reject(lambda: f(x, y.astype(np.float32)), TypeError, "float64")
    _reject(lambda: f(np.ones(N + 1)), ValueError, "shape")                                # wrong shape
    _reject(lambda: f(x, np.zeros((2, N))), ValueError, "shape")
    _reject(lambda: f(x, np.zeros(N)), ValueError, "shape")
    _reject(lambda: f(np.ones((2, 3, N))), ValueError, "shape")
    _reject(lambda: f(np.ones((3, 2 * N))[:, ::2]), ValueError, "contiguous")              # non-contiguous
    _reject(lambda: f(x, np.zeros((3, 2 * N))[:, ::2]), ValueError, "contiguous")
    _reject(lambda: f(x, beta=1.0), ValueError, "beta")                                     # y needed with beta != 0
    _reject(lambda: f(x, y, sigma=np.ones(2)), ValueError, "sigma")                         # one sigma per vector
    _reject(lambda: f(x, torch.zeros(3, N, dtype=torch.float64)), TypeError, "cannot be mixed")   # numpy / tensor mix
    _reject(lambda: f(torch.ones(3, N, dtype=torch.float64), y), TypeError, "cannot be mixed")
    tx, ty = torch.ones(3, N, dtype=torch.float64), torch.zeros(3, N, dtype=torch.float64)
    _reject(lambda: f(tx.float()), TypeError, "float64")
    _reject(lambda: f(tx, ty.float()), TypeError, "float64")
    _reject(lambda: f(tx, torch.zeros(3, 2 * N, dtype=torch.float64)[:, 1::2]), ValueError, "contiguous")
    _reject(lambda: f(tx, torch.zeros(4, N, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(tx, ty), TypeError, "CUDA")                                           # CPU tensors
    _reject(lambda: f(tx), TypeError, "CUDA")


def test_multiply_async_takes_cuda_tensors_only(B, dm):
    import torch
    f = dm.multiply_async
    tx, ty = torch.ones(3, N, dtype=torch.float64), torch.zeros(3, N, dtype=torch.float64)
    _reject(lambda: f(np.ones((3, N)), np.zeros((3, N))), TypeError, "CUDA tensors only")  # numpy
    _reject(lambda: f(tx, np.zeros((3, N))), TypeError, "CUDA tensors only")               # numpy / tensor mix
    _reject(lambda: f(tx, ty, sigma=np.ones(3)), TypeError, "CUDA tensors only")           # numpy sigma
    _reject(lambda: f(tx, None), TypeError, "CUDA tensors only")
    _reject(lambda: f(tx, ty), TypeError, "CUDA")                                           # CPU tensors
    _reject(lambda: f(tx.float(), ty), TypeError, "float64")
    _reject(lambda: f(tx, ty, sigma=torch.ones(3, dtype=torch.float32)), TypeError, "float64")
    _reject(lambda: f(tx, torch.zeros(2, N, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(tx, ty, sigma=torch.ones(2, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(torch.ones(3, 2 * N, dtype=torch.float64)[:, ::2], ty), ValueError, "contiguous")
    if torch.cuda.is_available():
        _reject(lambda: f(tx.cuda(), ty), TypeError, "CUDA")                                # CPU / CUDA mix
        _reject(lambda: f(tx.cuda(), ty.cuda(), sigma=torch.ones(3, dtype=torch.float64)), TypeError, "CUDA")
