"""CPU: the asynchronous solve's C ABI (bicg_solve_async, bicg_solve_async_prepare, bicg_matrix_history) is declared, exported and
bound, its bicg_result record has the layout of include/bicgstab_b200.h, and DeviceMatrix.solve_async rejects what it cannot use
before the library is called."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("bicg_solve_async", "bicg_solve_async_prepare", "bicg_matrix_history")


def test_async_symbols_declared_exported_and_bound(B):
    hdr = open(os.path.join(ROOT, "include", "bicgstab_b200.h")).read()
    out = subprocess.run(["nm", "-D", "--defined-only", B.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if l.strip()}
    for name in NEW:
        assert re.search(r"\bint\s+" + name + r"\s*\(", hdr), name
        assert name in exported, name
        assert name in B.SYMBOLS, name
        assert getattr(B.lib, name).restype is C.c_int


def test_bicg_result_layout(B):
    R = B._lib.bicg_result
    assert C.sizeof(R) == 24
    assert [getattr(R, f).offset for f in ("iters", "converged", "error", "reserved", "final_res")] == [0, 4, 8, 12, 16]
    src = open(os.path.join(ROOT, "mpi-bicgstab_b200", "csrc", "abi.cu")).read()
    assert "sizeof(bicg_result) == 24" in src and "offsetof(bicg_result, final_res) == 16" in src


def test_decode_result_reads_the_record(B):
    R = B._lib.bicg_result
    rec = R(iters=17, converged=1, error=0, reserved=0, final_res=3.5e-11)
    raw = np.frombuffer(bytes(rec), dtype=np.uint8)
    assert B.decode_result(raw) == {"iters": 17, "converged": 1, "error": 0, "final_res": 3.5e-11}
    with pytest.raises(ValueError):
        B.decode_result(raw[:16])


class _NoCall:
    """Stands in for the library: any call into it fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"the library was called ({name}) although the arguments were invalid")


def _bare_handle(B, n):
    dm = B.DeviceMatrix.__new__(B.DeviceMatrix)
    dm.blk = type("Blk", (), {"n_loc": n})()
    dm.h = None
    return dm


@pytest.fixture
def no_lib(B, monkeypatch):
    api = __import__(B.DeviceMatrix.__module__, fromlist=["lib"])
    monkeypatch.setattr(api, "lib", _NoCall())


def test_solve_async_rejects_numpy_wrong_dtype_and_non_contiguous(B, no_lib):
    torch = pytest.importorskip("torch")
    n = 8
    dm = _bare_handle(B, n)
    with pytest.raises(TypeError):
        dm.solve_async("bicgstab", np.zeros(n), np.ones(n))
    with pytest.raises(TypeError):
        dm.solve_async("bicgstab", torch.zeros(n, dtype=torch.float32), torch.ones(n, dtype=torch.float32))
    with pytest.raises(ValueError):
        dm.solve_async("bicgstab", torch.zeros(2 * n, dtype=torch.float64)[::2], torch.ones(n, dtype=torch.float64))
    with pytest.raises(ValueError):
        dm.solve_async("bicgstab", torch.zeros(n + 1, dtype=torch.float64), torch.ones(n + 1, dtype=torch.float64))
