"""CPU: the transpose in the C ABI -- bicg_matrix_create_transpose, bicg_matrix_transpose_values / _async and
bicg_matrix_block_nz are declared, exported and bound; a null handle or source, or a source that is not the transpose's, is
refused before the device is touched; the Python wrappers are there and check their source argument."""
import ctypes as C
import os

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTOS = ("bicg_matrix *bicg_matrix_create_transpose(bicg_matrix *m);",
          "int bicg_matrix_transpose_values(bicg_matrix *mt, bicg_matrix *src);",
          "int bicg_matrix_transpose_values_async(bicg_matrix *mt, bicg_matrix *src, void *stream);",
          "int bicg_matrix_block_nz(const bicg_matrix *m, unsigned *diag_nz, unsigned *offd_nz);")
NAMES = ("bicg_matrix_create_transpose", "bicg_matrix_transpose_values", "bicg_matrix_transpose_values_async",
         "bicg_matrix_block_nz")


def test_declared_exported_and_bound(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    exported = _exported(B)
    for proto, name in zip(PROTOS, NAMES):
        assert " ".join(proto.split()) in header, proto
        assert name in exported and name in B.SYMBOLS, name
    for meth in ("transpose", "transpose_values", "transpose_values_async"):
        assert callable(getattr(B.DeviceMatrix, meth)), meth


def _handle():
    """A zeroed stand-in for a handle: not a transpose (no source recorded), never used past the argument checks."""
    h = C.create_string_buffer(8192)
    return h, C.addressof(h)


def test_bad_arguments_without_gpu(B):
    """Null handles and a source that is not the transpose's return -1 (create: null) before the device is touched."""
    (h1, a), (h2, b) = _handle(), _handle()
    assert not B.lib.bicg_matrix_create_transpose(None)
    for mt, src in ((None, b), (a, None), (None, None), (a, b), (a, a)):
        assert B.lib.bicg_matrix_transpose_values(mt, src) == -1, (mt, src)
        assert B.lib.bicg_matrix_transpose_values_async(mt, src, None) == -1, (mt, src)
    d, o = C.c_uint(7), C.c_uint(7)
    assert B.lib.bicg_matrix_block_nz(None, C.byref(d), C.byref(o)) == -1
    assert B.lib.bicg_matrix_block_nz(a, None, C.byref(o)) == -1
    assert B.lib.bicg_matrix_block_nz(a, C.byref(d), None) == -1
    assert B.lib.bicg_matrix_block_nz(a, C.byref(d), C.byref(o)) == 0 and d.value == 0 and o.value == 0


N = 16


@pytest.fixture
def dm(B):
    """A DeviceMatrix of a one-rank block whose handle is a zeroed stand-in."""
    import scipy.sparse as sp
    A = sp.diags([-np.ones(N - 1), 4.0 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1], format="csr")
    blk = B.blocks_from_csr(N, A.indptr, A.indices, A.data)
    buf, addr = _handle()
    d = B.DeviceMatrix(blk, handle=addr)
    d._buf = buf
    yield d
    d.h = None


def test_wrappers_check_the_source(B, dm):
    with pytest.raises(TypeError, match="DeviceMatrix"):
        dm.transpose_values(np.zeros(N))
    with pytest.raises(TypeError, match="DeviceMatrix"):
        dm.transpose_values_async(None)
    with pytest.raises(ValueError, match="transpose_values failed with -1"):
        dm.transpose_values(dm)                      # the stand-in is not a transpose of anything


def test_handle_shape_for_set_values(B):
    """A transpose's DeviceMatrix has no host blocks: set_values checks against the counts the library reports."""
    shape = B.api._HandleShape(5, 9, 12, 3)
    assert (shape.n_loc, shape.n, shape.diag.nz, shape.offd.nz) == (5, 9, 12, 3)
    args = B.api._value_args(shape, np.zeros(12), np.zeros(3))
    assert [a[2] for a in args] == [(12,), (3,)]
