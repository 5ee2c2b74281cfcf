"""CPU: the value gradient in the C ABI -- bicg_matrix_value_grad and _async are declared, exported and bound; a null handle, u, v
or diag_out, nvec <= 0, a null offd_out on a handle with offd entries and an output overlapping u or v return -1 before the
device is touched; the Python wrappers (DeviceMatrix.value_grad / value_grad_async) reject bad arrays before they call the
library; importing the autograd module needs no GPU."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTOS = ("int bicg_matrix_value_grad(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, double beta, "
          "double *diag_out, double *offd_out, int device_vectors);",
          "int bicg_matrix_value_grad_async(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, "
          "double beta, double *diag_out, double *offd_out, void *stream);")
NAMES = ("bicg_matrix_value_grad", "bicg_matrix_value_grad_async")


def test_declared_exported_and_bound(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    exported = _exported(B)
    for proto, name in zip(PROTOS, NAMES):
        assert " ".join(proto.split()) in header, proto
        assert name in exported and name in B.SYMBOLS, name
    for meth in ("value_grad", "value_grad_async", "prepare_autograd"):
        assert callable(getattr(B.DeviceMatrix, meth)), meth


def _handle(n_loc, nnz, nnz_offd):
    """A zeroed stand-in for a handle, never used past the argument checks, with n_loc, nnz and nnz_offd set (the struct's
    third int and its two size_t after n_glob)."""
    h = C.create_string_buffer(8192)
    C.c_int.from_buffer(h, 8).value = n_loc
    C.c_size_t.from_buffer(h, 16).value = nnz
    C.c_size_t.from_buffer(h, 24).value = nnz_offd
    return h, C.addressof(h)


def test_bad_arguments_without_gpu(B):
    """Every -1 case returns before the device is touched, in both calls (the synchronous one for host and device pointers)."""
    buf = (C.c_double * 256)()
    base = C.addressof(buf)
    u, v, d, o = base, base + 8 * 32, base + 8 * 64, base + 8 * 128    # u, v: 2 x 4 doubles; diag 10, offd 6 entries
    calls = [lambda *a: B.lib.bicg_matrix_value_grad(*a, 0), lambda *a: B.lib.bicg_matrix_value_grad(*a, 1),
             lambda *a: B.lib.bicg_matrix_value_grad_async(*a, None)]
    h, hp = _handle(4, 16, 6)
    h1, hp1 = _handle(4, 10, 0)                                        # no offd entries
    for call in calls:
        for args in ((None, 2, u, v, d, o), (hp, 2, None, v, d, o), (hp, 2, u, None, d, o), (hp, 2, u, v, None, o),  # nulls
                     (hp, 0, u, v, d, o), (hp, -1, u, v, d, o),                                   # nvec <= 0
                     (hp, 2, u, v, d, None),                                                      # offd entries, no offd_out
                     (hp, 2, u, v, u, o), (hp, 2, u, v, d, v + 8 * 7), (hp, 2, u, v, u + 8 * 7, o),  # overlaps
                     (hp, 2, u, v, v - 8 * 9, o), (hp1, 2, u, v, u - 8 * 9, None)):
            assert call(args[0], args[1], args[2], args[3], 1.0, 0.0, args[4], args[5]) == -1, args


@pytest.mark.parametrize("call", ["B.lib.bicg_matrix_value_grad(hp, 2, u, v, -1.0, 0.0, d, None, 0)",
                                  "B.lib.bicg_matrix_value_grad_async(hp, 2, u, v, 1.0, 0.5, d, None, None)"])
def test_valid_call_fails_loudly_without_gpu(B, call):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys, ctypes as C; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; "
            "h = C.create_string_buffer(8192); C.c_int.from_buffer(h, 8).value = 4; C.c_size_t.from_buffer(h, 16).value = 10; "
            "hp = C.addressof(h); b = (C.c_double * 256)(); u = C.addressof(b); v = u + 8 * 32; d = u + 8 * 64; "
            "%s; print('RETURNED')" % (ROOT, call))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


# ---- the Python wrappers reject bad arrays before the library sees them --------------------------------------------------
N = 64


@pytest.fixture
def dm(B):
    """A DeviceMatrix of a one-rank tridiagonal block (3 N - 2 diag entries) whose handle is never used."""
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


def test_value_grad_rejects_bad_arrays(B, dm):
    import torch
    f = dm.value_grad
    nz = 3 * N - 2
    u, v = np.ones((3, N)), np.ones((3, N))
    _reject(lambda: f(u.astype(np.float32), v), TypeError, "float64")
    _reject(lambda: f(u, v.astype(np.float32)), TypeError, "float64")
    _reject(lambda: f(u, np.ones((2, N))), ValueError, "shape")                              # u, v disagree
    _reject(lambda: f(np.ones(N + 1), np.ones(N + 1)), ValueError, "shape")
    _reject(lambda: f(u, v, diag_out=np.zeros(nz + 1)), ValueError, "shape")                 # wrong output length
    _reject(lambda: f(u, v, diag_out=np.zeros(2 * nz)[::2]), ValueError, "contiguous")
    _reject(lambda: f(u, v, beta=1.0), ValueError, "beta")                                   # outputs needed with beta != 0
    _reject(lambda: f(u, torch.ones(3, N, dtype=torch.float64)), TypeError, "cannot be mixed")
    _reject(lambda: f(u, v, diag_out=torch.zeros(nz, dtype=torch.float64)), TypeError, "cannot be mixed")
    tu = torch.ones(3, N, dtype=torch.float64)
    _reject(lambda: f(tu, tu.clone()), TypeError, "CUDA")                                    # CPU tensors


def test_value_grad_async_takes_cuda_tensors_only(B, dm):
    import torch
    f = dm.value_grad_async
    tu = torch.ones(3, N, dtype=torch.float64)
    _reject(lambda: f(np.ones((3, N)), np.ones((3, N))), TypeError, "CUDA tensors only")
    _reject(lambda: f(tu, np.ones((3, N))), TypeError, "CUDA tensors only")
    _reject(lambda: f(tu, tu, diag_out=np.zeros(3 * N - 2)), TypeError, "CUDA tensors only")
    _reject(lambda: f(tu, tu.clone(), beta=2.0), ValueError, "beta")
    _reject(lambda: f(tu.float(), tu), TypeError, "float64")
    _reject(lambda: f(tu, torch.ones(2, N, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(tu, tu.clone()), TypeError, "CUDA")


def test_autograd_imports_without_gpu(B):
    """The package does not import torch; its autograd entry points load on first use, with no GPU needed."""
    code = ("import sys; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; assert 'torch' not in sys.modules; "
            "f = B.solve_autograd; g = B.multiply_autograd; import torch; "
            "assert issubclass(B.SolveFunction, torch.autograd.Function) and issubclass(B.MultiplyFunction, torch.autograd.Function); "
            "print('AUTOGRAD_OK')" % ROOT)
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert p.returncode == 0 and "AUTOGRAD_OK" in p.stdout, p.stderr


def test_autograd_rejects_bad_inputs_without_gpu(B, dm):
    import torch
    _reject(lambda: B.solve_autograd(dm, np.ones(N)), TypeError, "CUDA float64 tensor")
    _reject(lambda: B.multiply_autograd(dm, np.ones(N)), TypeError, "CUDA float64 tensor")
    _reject(lambda: B.solve_autograd(dm, torch.ones(N + 1, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: B.solve_autograd(dm, torch.ones(N, dtype=torch.float32)), TypeError, "float64")
    _reject(lambda: B.multiply_autograd(dm, torch.ones(N, dtype=torch.float64)), TypeError, "CUDA")
    _reject(lambda: B.solve_autograd(dm, torch.ones(N, dtype=torch.float64), offd_val=torch.ones(3, dtype=torch.float64)),
            ValueError, "without diag_val")                                                 # offd values alone
    _reject(lambda: B.multiply_autograd(dm, torch.ones(N, dtype=torch.float64), offd_val=torch.ones(3, dtype=torch.float64)),
            ValueError, "without diag_val")


def test_value_grad_layout_hook_rejects_bad_arguments(B):
    """bicg_debug_value_grad_layout: a null handle, a group width that is no power of two up to 32, and split rows on a handle
    with offd entries are refused"""
    buf = C.create_string_buffer(8192)
    h = C.addressof(buf)
    blk = (C.c_uint * 8)()
    assert B.lib.bicg_debug_value_grad_layout(None, 0, None) == -1
    for lanes in (-1, 3, 6, 64):
        assert B.lib.bicg_debug_value_grad_layout(h, lanes, None) == -1, lanes
    assert B.lib.bicg_debug_value_grad_layout(h, 16, blk) == 0
    assert B.lib.bicg_debug_value_grad_layout(h, 0, None) == 0
    C.c_size_t.from_buffer(buf, 24).value = 5                      # offd entries
    assert B.lib.bicg_debug_value_grad_layout(h, 0, blk) == -1
