"""CPU: new values on a resident matrix in the C ABI -- bicg_matrix_set_values, _async and bicg_matrix_shift_diagonal are declared,
exported and bound, a null handle or null diag_val returns -1 before the device is touched, a valid call without a GPU exits 1,
and the Python wrappers (DeviceMatrix.set_values / set_values_async) reject bad arrays before they call the library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTOS = ("int bicg_matrix_set_values(bicg_matrix *m, const double *diag_val, const double *offd_val, int device_vectors);",
          "int bicg_matrix_set_values_async(bicg_matrix *m, const double *diag_val, const double *offd_val, void *stream);",
          "int bicg_matrix_shift_diagonal(bicg_matrix *m, double sigma);")
NAMES = ("bicg_matrix_set_values", "bicg_matrix_set_values_async", "bicg_matrix_shift_diagonal")


def test_declared_exported_and_bound(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    exported = _exported(B)
    for proto, name in zip(PROTOS, NAMES):
        assert " ".join(proto.split()) in header, proto
        assert name in exported and name in B.SYMBOLS, name


def test_null_handle_or_values_without_gpu(B):
    """A null handle or null diag_val returns -1 before the device is touched (the handle is a zeroed buffer, never read)."""
    h = C.create_string_buffer(64)
    hp = C.addressof(h)
    d = (C.c_double * 4)()
    o = (C.c_double * 4)()
    for dev in (0, 1):
        assert B.lib.bicg_matrix_set_values(None, d, o, dev) == -1
        assert B.lib.bicg_matrix_set_values(hp, None, o, dev) == -1
        assert B.lib.bicg_matrix_set_values(hp, None, None, dev) == -1
    assert B.lib.bicg_matrix_set_values_async(None, d, o, None) == -1
    assert B.lib.bicg_matrix_set_values_async(hp, None, o, None) == -1
    assert B.lib.bicg_matrix_shift_diagonal(None, 0.5) == -1


@pytest.mark.parametrize("call", ["B.lib.bicg_matrix_set_values(hp, d, None, 0)",
                                  "B.lib.bicg_matrix_set_values_async(hp, d, None, None)",
                                  "B.lib.bicg_matrix_shift_diagonal(hp, 0.5)"])
def test_valid_call_fails_loudly_without_gpu(B, call):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys, ctypes as C; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; "
            "h = C.create_string_buffer(4096); hp = C.addressof(h); d = (C.c_double * 8)(); "
            "%s; print('RETURNED')" % (ROOT, call))
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


# ---- the Python wrappers reject bad values before the library sees them ----------------------------------------------------
@pytest.fixture
def dm(B):
    """A DeviceMatrix of a two-rank block split (rank 0 of 2: diag and offd entries) whose handle is never used."""
    import scipy.sparse as sp
    n = 64
    A = sp.diags([-np.ones(n - 8), -np.ones(n - 1), 6.0 * np.ones(n), -np.ones(n - 1), -np.ones(n - 8)], [-8, -1, 0, 1, 8],
                 format="csr")
    blk = B.blocks_from_csr(n, A.indptr, A.indices, A.data, rank=0, world=2)
    assert int(blk.diag.nz) > 0 and int(blk.offd.nz) == 9
    d = B.DeviceMatrix.__new__(B.DeviceMatrix)
    d.blk, d.h = blk, None
    yield d
    d.h = None


def _reject(fn, exc, text):
    with pytest.raises(exc, match=text):
        fn()


def test_set_values_rejects_bad_arrays(B, dm):
    import torch
    nd, no = int(dm.blk.diag.nz), int(dm.blk.offd.nz)
    dv, ov = np.ones(nd), np.ones(no)
    f = dm.set_values
    _reject(lambda: f(dv.astype(np.float32), ov), TypeError, "float64")                 # wrong dtype
    _reject(lambda: f(dv, ov.astype(np.int64)), TypeError, "float64")
    _reject(lambda: f(np.ones(nd + 1), ov), ValueError, "shape")                        # wrong length
    _reject(lambda: f(dv, np.ones(no - 1)), ValueError, "shape")
    _reject(lambda: f(np.ones((nd, 1)), ov), ValueError, "shape")
    _reject(lambda: f(np.ones(2 * nd)[::2], ov), ValueError, "contiguous")              # non-contiguous
    _reject(lambda: f(dv, torch.ones(no, dtype=torch.float64)), TypeError, "cannot be mixed")   # numpy / tensor mix
    _reject(lambda: f(torch.ones(nd, dtype=torch.float64), ov), TypeError, "cannot be mixed")
    td, to = torch.ones(nd, dtype=torch.float64), torch.ones(no, dtype=torch.float64)
    _reject(lambda: f(td.float(), to), TypeError, "float64")
    _reject(lambda: f(td, torch.ones(2 * no, dtype=torch.float64)[1::2]), ValueError, "contiguous")
    _reject(lambda: f(td, torch.ones(no + 1, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(td, to), TypeError, "CUDA")                                        # CPU tensors


def test_offd_values_required_with_several_ranks(B, dm, monkeypatch):
    """None stands for an empty offd block only: with several ranks a block with offd entries needs them."""
    class _Lib:
        def __getattr__(self, name):
            return getattr(B.lib, name)

        @staticmethod
        def bicg_comm_world():
            return 2
    import sys
    monkeypatch.setattr(sys.modules[B.DeviceMatrix.__module__], "lib", _Lib())
    _reject(lambda: dm.set_values(np.ones(int(dm.blk.diag.nz))), ValueError, "offd_val")


def test_set_values_async_takes_cuda_tensors_only(B, dm):
    import torch
    nd, no = int(dm.blk.diag.nz), int(dm.blk.offd.nz)
    f = dm.set_values_async
    td, to = torch.ones(nd, dtype=torch.float64), torch.ones(no, dtype=torch.float64)
    _reject(lambda: f(np.ones(nd), np.ones(no)), TypeError, "CUDA tensors only")        # numpy
    _reject(lambda: f(td, np.ones(no)), TypeError, "CUDA tensors only")                  # numpy / tensor mix
    _reject(lambda: f(td, to), TypeError, "CUDA")                                        # CPU tensors
    _reject(lambda: f(td.float(), to), TypeError, "float64")
    _reject(lambda: f(td, torch.ones(no - 1, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(torch.ones(2 * nd, dtype=torch.float64)[::2], to), ValueError, "contiguous")
    if torch.cuda.is_available():
        _reject(lambda: f(td.cuda(), to), TypeError, "CUDA")                             # CPU / CUDA mix
