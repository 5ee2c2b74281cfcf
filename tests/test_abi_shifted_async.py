"""CPU: the asynchronous shifted solve's C ABI (bicg_shifted_solve_async, bicg_shifted_solve_async_prepare,
bicg_matrix_shift_history) is declared, exported and bound, its bicg_shift_result record has the layout of
include/bicgstab_b200.h, decode_shift_result reads it, and DeviceMatrix.shifted_solve_async rejects what it cannot use before the
library is called."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("bicg_shifted_solve_async", "bicg_shifted_solve_async_prepare", "bicg_matrix_shift_history")
FIELDS = ("ret", "iters", "converged", "seed", "error", "reserved", "final_res")


def test_shifted_async_symbols_declared_exported_and_bound(B):
    hdr = open(os.path.join(ROOT, "include", "bicgstab_b200.h")).read()
    out = subprocess.run(["nm", "-D", "--defined-only", B.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if l.strip()}
    for name in NEW:
        assert re.search(r"\bint\s+" + name + r"\s*\(", hdr), name
        assert name in exported, name
        assert name in B.SYMBOLS, name
        assert getattr(B.lib, name).restype is C.c_int
    assert len(B.SYMBOLS["bicg_shifted_solve_async"][1]) == 10
    assert len(B.SYMBOLS["bicg_shifted_solve_async_prepare"][1]) == 3


def test_bicg_shift_result_layout(B):
    R = B._lib.bicg_shift_result
    assert C.sizeof(R) == 32
    assert [getattr(R, f).offset for f in FIELDS] == [0, 4, 8, 12, 16, 20, 24]
    hdr = open(os.path.join(ROOT, "include", "bicgstab_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} bicg_shift_result;", hdr).group(1)
    assert re.findall(r"\b(\w+);", body) == list(FIELDS)
    src = open(os.path.join(ROOT, "mpi-bicgstab_b200", "csrc", "abi.cu")).read()
    assert "sizeof(bicg_shift_result) == 32" in src
    for f, off in zip(FIELDS, [0, 4, 8, 12, 16, 20, 24]):
        assert f"offsetof(bicg_shift_result, {f}) == {off}" in src, f


def test_decode_shift_result_reads_the_record(B):
    R = B._lib.bicg_shift_result
    rec = R(ret=42, iters=41, converged=1, seed=3, error=0, reserved=0, final_res=2.25e-13)
    raw = np.frombuffer(bytes(rec), dtype=np.uint8)
    assert B.decode_shift_result(raw) == {"ret": 42, "iters": 41, "converged": 1, "seed": 3, "error": 0, "final_res": 2.25e-13}
    with pytest.raises(ValueError):
        B.decode_shift_result(raw[:24])
    with pytest.raises(ValueError):                       # a plain solve's record is not a shifted one
        B.decode_shift_result(np.frombuffer(bytes(B._lib.bicg_result()), dtype=np.uint8))


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


def test_shifted_solve_async_rejects_bad_arguments(B, no_lib):
    torch = pytest.importorskip("torch")
    n, L = 8, 3
    dm = _bare_handle(B, n)
    f64 = dict(dtype=torch.float64)
    x, r, sg = torch.zeros(L, n, **f64), torch.ones(n, **f64), torch.arange(L, **f64) * 0.01
    m = "shifted_lopbicgstab"
    with pytest.raises(TypeError):                        # numpy vectors
        dm.shifted_solve_async(m, np.zeros((L, n)), np.ones(n), sg, 0)
    with pytest.raises(TypeError):                        # host sigma as numpy
        dm.shifted_solve_async(m, x, r, np.arange(L) * 0.01, 0)
    with pytest.raises(TypeError):                        # CPU tensors, sigma included
        dm.shifted_solve_async(m, x, r, sg, 0)
    with pytest.raises(TypeError):                        # float32
        dm.shifted_solve_async(m, x.float(), r.float(), sg.float(), 0)
    with pytest.raises(ValueError):                       # x_set of the wrong shape
        dm.shifted_solve_async(m, torch.zeros(L + 1, n, **f64), r, sg, 0)
    with pytest.raises(ValueError):                       # r of the wrong length
        dm.shifted_solve_async(m, x, torch.ones(n + 1, **f64), sg, 0)
    with pytest.raises(ValueError):                       # non-contiguous x_set
        dm.shifted_solve_async(m, torch.zeros(n, L, **f64).t(), r, sg, 0)
    with pytest.raises(ValueError):                       # 2-d sigma
        dm.shifted_solve_async(m, x, r, sg.view(1, L), 0)
    for seed in (-1, L, 1.0, True, None):
        with pytest.raises(ValueError):
            dm.shifted_solve_async(m, x, r, sg, seed)
