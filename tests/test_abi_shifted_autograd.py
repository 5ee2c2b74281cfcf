"""CPU: the pieces of a differentiable shifted solve in the C ABI -- bicg_matrix_shift_diagonal_async, its prepare step and
bicg_matrix_dots_async are declared, exported and bound; every -1 case returns before the device is touched and valid calls fail
loudly without a GPU; the Python wrappers (DeviceMatrix.shift_diagonal_async, dots_async) and shifted_solve_autograd reject
bad arrays before they call the library; shifted_solve_autograd loads on first use without the package importing torch."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTOS = ("int bicg_matrix_shift_diagonal_async(bicg_matrix *m, const double *sigma, void *stream);",
          "int bicg_matrix_shift_diagonal_async_prepare(bicg_matrix *m);",
          "int bicg_matrix_dots_async(bicg_matrix *m, int nvec, const double *u, const double *v, double *out, void *stream);")
NAMES = ("bicg_matrix_shift_diagonal_async", "bicg_matrix_shift_diagonal_async_prepare", "bicg_matrix_dots_async")


def test_declared_exported_and_bound(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    exported = _exported(B)
    for proto, name in zip(PROTOS, NAMES):
        assert " ".join(proto.split()) in header, proto
        assert name in exported and name in B.SYMBOLS, name
    for meth in ("shift_diagonal_async", "prepare_shift_diagonal_async", "dots_async", "prepare_shifted_autograd"):
        assert callable(getattr(B.DeviceMatrix, meth)), meth


def test_bad_arguments_without_gpu(B):
    """A null handle, sigma, u, v or out, and nvec <= 0, return -1 before the device is touched"""
    h = C.create_string_buffer(8192)
    hp = C.addressof(h)
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    assert B.lib.bicg_matrix_shift_diagonal_async(None, p, None) == -1
    assert B.lib.bicg_matrix_shift_diagonal_async(hp, None, None) == -1
    assert B.lib.bicg_matrix_shift_diagonal_async_prepare(None) == -1
    for args in ((None, 1, p, p + 64, p + 128), (hp, 1, None, p, p + 128), (hp, 1, p, None, p + 128), (hp, 1, p, p + 64, None),
                 (hp, 0, p, p + 64, p + 128), (hp, -3, p, p + 64, p + 128)):
        assert B.lib.bicg_matrix_dots_async(*args, None) == -1, args


@pytest.mark.parametrize("call", ["B.lib.bicg_matrix_shift_diagonal_async(hp, p, None)",
                                  "B.lib.bicg_matrix_shift_diagonal_async_prepare(hp)",
                                  "B.lib.bicg_matrix_dots_async(hp, 2, p, p + 64, p + 128, None)"])
def test_valid_call_fails_loudly_without_gpu(B, call):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys, ctypes as C; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; "
            "h = C.create_string_buffer(8192); C.c_int.from_buffer(h, 8).value = 4; hp = C.addressof(h); "
            "b = (C.c_double * 64)(); p = C.addressof(b); %s; print('RETURNED')" % (ROOT, call))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


# ---- the Python wrappers reject bad arrays before the library sees them --------------------------------------------------
N = 64


@pytest.fixture
def dm(B):
    """A DeviceMatrix of a one-rank tridiagonal block whose handle is never used."""
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


def test_shift_diagonal_async_rejects_bad_sigma(B, dm):
    import torch
    f = dm.shift_diagonal_async
    _reject(lambda: f(0.5), TypeError, "CUDA tensor")
    _reject(lambda: f(np.ones(1)), TypeError, "CUDA tensor")
    _reject(lambda: f(torch.ones(1, dtype=torch.float32)), TypeError, "float64")
    _reject(lambda: f(torch.ones(2, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(torch.ones((), dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(torch.ones(4, dtype=torch.float64)[::2][:1].expand(1)), TypeError, "CUDA")   # CPU tensor


def test_dots_async_rejects_bad_arrays(B, dm):
    import torch
    f = dm.dots_async
    tu = torch.ones(3, N, dtype=torch.float64)
    _reject(lambda: f(np.ones((3, N)), np.ones((3, N))), TypeError, "CUDA tensors only")
    _reject(lambda: f(tu, np.ones((3, N))), TypeError, "CUDA tensors only")
    _reject(lambda: f(tu, tu, out=np.zeros(3)), TypeError, "CUDA tensors only")
    _reject(lambda: f(tu.float(), tu), TypeError, "float64")
    _reject(lambda: f(tu, torch.ones(2, N, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(tu, tu.clone(), out=torch.zeros(4, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(tu, torch.ones(3, 2 * N, dtype=torch.float64)[:, ::2]), ValueError, "contiguous")
    _reject(lambda: f(tu, tu.clone()), TypeError, "CUDA")                                  # CPU tensors


def test_shifted_autograd_rejects_bad_inputs_without_gpu(B, dm):
    import torch
    b, s = torch.ones(N, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    f = B.shifted_solve_autograd
    _reject(lambda: f(dm, b, np.zeros(3)), TypeError, "CUDA float64 tensor")
    _reject(lambda: f(dm, b, torch.zeros(1, 3, dtype=torch.float64)), ValueError, "1-d")
    _reject(lambda: f(dm, b, torch.zeros((), dtype=torch.float64)), ValueError, "1-d")
    _reject(lambda: f(dm, torch.ones(N + 1, dtype=torch.float64), s), ValueError, "shape")
    _reject(lambda: f(dm, torch.ones(2, N, dtype=torch.float64), s), ValueError, "shape")
    _reject(lambda: f(dm, b, s.float()), TypeError, "float64")
    _reject(lambda: f(dm, b, s, x0=torch.zeros(2, N, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(dm, b, s, offd_val=torch.ones(3, dtype=torch.float64)), ValueError, "without diag_val")
    _reject(lambda: f(dm, b, s), TypeError, "CUDA")                                          # CPU tensors
    _reject(lambda: B.multiply_autograd(dm, b, sigma=np.zeros(1)), TypeError, "CUDA")


def test_shifted_autograd_loads_on_first_use_without_gpu(B):
    """The package does not import torch; shifted_solve_autograd loads with the autograd module on first use."""
    code = ("import sys; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; assert 'torch' not in sys.modules; "
            "f = B.shifted_solve_autograd; import torch; assert issubclass(B.ShiftedSolveFunction, torch.autograd.Function); "
            "print('SHIFTED_AUTOGRAD_OK')" % ROOT)
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert p.returncode == 0 and "SHIFTED_AUTOGRAD_OK" in p.stdout, p.stderr
