"""CPU: the two entry points a differentiable backward is built from -- bicg_matrix_multiply_values_async (and its prepare) and
bicg_matrix_transpose_entries_async -- are declared, exported and bound; their -1 cases return before the device is touched;
the Python wrappers (DeviceMatrix.multiply_values_async / transpose_entries_async) reject bad tensors before they call the
library; the autograd module, whose Functions are now all differentiable, imports without a GPU."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTOS = ("int bicg_matrix_multiply_values_async(bicg_matrix *m, int nvec, const double *w_diag, const double *w_offd, "
          "const double *x, double *y, double alpha, double beta, void *stream);",
          "int bicg_matrix_multiply_values_async_prepare(bicg_matrix *m);",
          "int bicg_matrix_transpose_entries_async(bicg_matrix *mt, bicg_matrix *src, int reverse, const double *in_diag, "
          "const double *in_offd, double *out_diag, double *out_offd, void *stream);")
NAMES = ("bicg_matrix_multiply_values_async", "bicg_matrix_multiply_values_async_prepare", "bicg_matrix_transpose_entries_async")


def test_declared_exported_and_bound(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    exported = _exported(B)
    for proto, name in zip(PROTOS, NAMES):
        assert " ".join(proto.split()) in header, proto
        assert name in exported and name in B.SYMBOLS, name
    for meth in ("multiply_values_async", "prepare_multiply_values_async", "transpose_entries_async"):
        assert callable(getattr(B.DeviceMatrix, meth)), meth


def _handle(n_loc, nnz, nnz_offd):
    """A zeroed stand-in for a handle (never a transpose), with n_loc, nnz and nnz_offd set"""
    h = C.create_string_buffer(8192)
    C.c_int.from_buffer(h, 8).value = n_loc
    C.c_size_t.from_buffer(h, 16).value = nnz
    C.c_size_t.from_buffer(h, 24).value = nnz_offd
    return h, C.addressof(h)


def test_multiply_values_bad_arguments_without_gpu(B):
    buf = (C.c_double * 256)()
    base = C.addressof(buf)
    x, y, wd, wo = base, base + 8 * 32, base + 8 * 64, base + 8 * 128   # x, y: 2 x 4 doubles; W: 10 diag, 6 offd entries
    h, hp = _handle(4, 16, 6)
    h1, hp1 = _handle(4, 10, 0)
    f = B.lib.bicg_matrix_multiply_values_async
    for args in ((None, 2, wd, wo, x, y), (hp, 2, None, wo, x, y), (hp, 2, wd, wo, None, y), (hp, 2, wd, wo, x, None),  # nulls
                 (hp, 0, wd, wo, x, y), (hp, -1, wd, wo, x, y),                                    # nvec <= 0
                 (hp, 2, wd, None, x, y),                                                          # offd entries, no w_offd
                 (hp, 2, wd, wo, x, x + 8 * 7), (hp, 2, wd, wo, y, y),                             # x overlaps y
                 (hp, 2, y + 8 * 7, wo, x, y), (hp, 2, wd, y - 8 * 5, x, y),                       # W overlaps y
                 (hp1, 2, y - 8 * 9, None, x, y)):
        assert f(args[0], args[1], args[2], args[3], args[4], args[5], 1.0, 0.0, None) == -1, args
    assert B.lib.bicg_matrix_multiply_values_async_prepare(None) == -1


def test_transpose_entries_bad_arguments_without_gpu(B):
    """null handles, reverse outside {0, 1}, null or overlapping vectors, a missing offd vector and a handle that is not a
    transpose of the other return -1 before the device is touched.  The stand-ins are never a transpose, so every call here is
    refused; test_gpu_second_order.py checks each case on a real pair, where the valid call succeeds."""
    buf = (C.c_double * 64)()
    i, o = C.addressof(buf), C.addressof(buf) + 8 * 32
    (h1, a), (h2, b) = _handle(4, 10, 0), _handle(4, 10, 0)
    (h3, c), = (_handle(4, 12, 2),)
    f = B.lib.bicg_matrix_transpose_entries_async
    for mt, src, rev, ind, ino, outd in ((None, b, 0, i, None, o), (a, None, 0, i, None, o), (a, b, 0, i, None, o),
                                         (a, a, 1, i, None, o), (a, b, 2, i, None, o), (a, b, -1, i, None, o),
                                         (a, b, 0, None, None, o), (a, b, 0, i, None, None), (a, b, 1, i, None, i),
                                         (a, b, 0, i, None, i + 8 * 9), (a, c, 0, i, None, o), (a, c, 0, i, o + 8 * 12, o)):
        assert f(mt, src, rev, ind, ino, outd, None, None) == -1, (mt, src, rev)


N = 16


@pytest.fixture
def dms(B):
    """(dm, mt): DeviceMatrix objects of a one-rank tridiagonal block whose handles are zeroed stand-ins, mt linked as dm's
    transpose"""
    import scipy.sparse as sp
    A = sp.diags([-np.ones(N - 1), 4.0 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1], format="csr")
    bufs = [C.create_string_buffer(8192) for _ in range(2)]
    dm = B.DeviceMatrix(B.blocks_from_csr(N, A.indptr, A.indices, A.data), handle=C.addressof(bufs[0]))
    mt = B.DeviceMatrix(B.blocks_from_csr(N, A.indptr, A.indices, A.data), handle=C.addressof(bufs[1]))
    dm._t, mt._src, dm._bufs = mt, dm, bufs
    yield dm, mt
    dm.h = mt.h = None
    dm._t = mt._src = None


def _reject(fn, exc, text):
    with pytest.raises(exc, match=text):
        fn()


def test_multiply_values_wrapper_rejects_bad_tensors(B, dms):
    import torch
    dm, _ = dms
    f = dm.multiply_values_async
    nz = 3 * N - 2
    w, x = torch.ones(nz, dtype=torch.float64), torch.ones(3, N, dtype=torch.float64)
    _reject(lambda: f(np.ones(nz), None, x), TypeError, "CUDA float64 tensor")
    _reject(lambda: f(w, None, np.ones((3, N))), TypeError, "CUDA tensors only")
    _reject(lambda: f(w, None, x, np.ones((3, N))), TypeError, "CUDA tensors only")
    _reject(lambda: f(w, None, x, beta=1.0), ValueError, "beta")
    _reject(lambda: f(w.float(), None, x), TypeError, "float64")
    _reject(lambda: f(torch.ones(nz + 1, dtype=torch.float64), None, x), ValueError, "shape")
    _reject(lambda: f(w, None, x, torch.ones(2, N, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(torch.ones(2 * nz, dtype=torch.float64)[::2], None, x), ValueError, "contiguous")
    _reject(lambda: f(w, None, x), TypeError, "CUDA")                                        # CPU tensors


def test_transpose_entries_wrapper_rejects_bad_tensors(B, dms):
    import torch
    dm, mt = dms
    nz = 3 * N - 2
    r = torch.ones(nz, dtype=torch.float64)
    _reject(lambda: mt.transpose_entries_async(None, r), TypeError, "DeviceMatrix")
    _reject(lambda: mt.transpose_entries_async(dm, np.ones(nz)), TypeError, "CUDA float64 tensor")
    _reject(lambda: mt.transpose_entries_async(dm, torch.ones(nz + 1, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: mt.transpose_entries_async(dm, r.float()), TypeError, "float64")
    _reject(lambda: mt.transpose_entries_async(dm, r, out=r), TypeError, "pair")
    _reject(lambda: mt.transpose_entries_async(dm, r, out=(torch.ones(nz - 1, dtype=torch.float64), None)), ValueError, "shape")
    _reject(lambda: mt.transpose_entries_async(dm, r, reverse=True), TypeError, "CUDA")      # CPU tensors


def test_back_link_is_not_owned(B, dms):
    """the adjoint of a linked transpose is its source; destroying the transpose leaves the source alone"""
    dm, mt = dms
    assert dm._adjoint() is mt and mt._adjoint() is dm
    mt.h = None                                      # nothing to free: the stand-in is not a library handle
    mt.destroy()
    assert dm.h is not None and mt._src is None


def test_autograd_imports_without_gpu(B):
    """Every Function is differentiable (no once_differentiable wrapper), and the module loads with no GPU."""
    code = ("import sys; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; import torch; "
            "import mpi_bicgstab_b200.autograd as A; "
            "fs = [A.SolveFunction, A.ShiftedSolveFunction, A.MultiplyFunction, A._ValueGrad, A._MultiplyValues, A._Dots, "
            "A._TransposeEntries]; "
            "assert all(issubclass(f, torch.autograd.Function) for f in fs); "
            "assert all('once_differentiable' not in repr(f.backward) for f in fs); "
            "assert not hasattr(A, 'once_differentiable'); print('AUTOGRAD_OK')" % ROOT)
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert p.returncode == 0 and "AUTOGRAD_OK" in p.stdout, p.stderr
