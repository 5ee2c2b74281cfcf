"""CPU: the shifted solvers on device vectors in the C ABI -- bicg_shifted_solve_dev is declared and exported, its argument check
runs before the device check and is collective over the ranks, a valid call without a GPU exits 1, and the Python wrappers
(DeviceMatrix.shifted_solve / DeviceMatrix.solve) reject bad tensors before they call the library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_abi import ROOT, _exported

PROTO = ("int bicg_shifted_solve_dev(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, "
         "int seed,")


def test_declared_and_exported(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = " ".join(f.read().split())
    assert " ".join(PROTO.split()) in header
    assert "bicg_shifted_solve_dev" in _exported(B) and "bicg_shifted_solve_dev" in B.SYMBOLS
    assert "shifted_bicgstab" not in _exported(B)


def test_rejects_bad_arguments_without_gpu(B):
    """Every invalid argument returns -1 before the device is touched (the handle is a zeroed buffer, never read)."""
    h = C.create_string_buffer(64)
    x = (C.c_double * 8)(); r = (C.c_double * 4)(); s = (C.c_double * 2)(0.1, 0.2)
    st = B.bicg_stats()
    f = B.lib.bicg_shifted_solve_dev
    hp = C.addressof(h)
    assert f(None, 0, x, r, s, 2, 0, C.byref(st)) == -1                   # null handle
    assert f(hp, 0, None, r, s, 2, 0, C.byref(st)) == -1                  # null x_set
    assert f(hp, 0, x, None, s, 2, 0, C.byref(st)) == -1                  # null r
    assert f(hp, 0, x, r, None, 2, 0, C.byref(st)) == -1                  # null sigma
    for method in (-1, 4, 99):                                             # unknown method
        assert f(hp, method, x, r, s, 2, 0, C.byref(st)) == -1
    assert f(hp, 0, x, r, s, 0, 0, C.byref(st)) == -1                     # sigma_len <= 0
    assert f(hp, 0, x, r, s, -3, 0, C.byref(st)) == -1
    for seed in (-1, 2, 5):                                                # seed outside [0, sigma_len)
        assert f(hp, 1, x, r, s, 2, seed, C.byref(st)) == -1


def test_valid_call_fails_loudly_without_gpu(B):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys, ctypes as C; sys.path.insert(0, %r); import mpi_bicgstab_b200 as B; "
            "h = C.create_string_buffer(4096); x = (C.c_double * 8)(); r = (C.c_double * 4)(); s = (C.c_double * 2)(0.1, 0.2); "
            "B.lib.bicg_shifted_solve_dev(C.addressof(h), 1, x, r, s, 2, 1, None); print('RETURNED')" % ROOT)
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


_COLLECTIVE_C = r"""
#include <stdio.h>
#include "bicgstab_b200.h"
int bicg_shm_bootstrap(void); void bicg_shm_shutdown(void);
int main(void)
{
    bicg_shm_bootstrap();
    const int rank = bicg_comm_rank();
    static char handle[4096];                       /* never read: every call below fails its collective argument check */
    double x[8] = {0}, r[4] = {1, 1, 1, 1}, s[3] = {0.1, 0.2, 0.3};
    bicg_stats st;
    int v[7];
    v[0] = bicg_shifted_solve_dev((bicg_matrix *)handle, 1, rank == 1 ? NULL : x, r, s, 2, 0, &st);  /* one rank: null x_set */
    v[1] = bicg_shifted_solve_dev((bicg_matrix *)handle, 1, x, r, s, 2, rank == 2 ? 2 : 0, &st);     /* one rank: bad seed */
    v[2] = bicg_shifted_solve_dev((bicg_matrix *)handle, rank == 0 ? 7 : 1, x, r, s, 2, 0, &st);     /* one rank: bad method */
    v[3] = bicg_shifted_solve_dev((bicg_matrix *)handle, 1, x, r, s, rank == 2 ? 3 : 2, 0, &st);     /* sigma_len differs */
    v[4] = bicg_shifted_solve_dev((bicg_matrix *)handle, 1, x, r, s, 3, rank == 1 ? 1 : 0, &st);     /* seed differs */
    v[5] = bicg_shifted_solve_dev((bicg_matrix *)handle, rank == 2 ? 2 : 1, x, r, s, 2, 0, &st);     /* method differs */
    v[6] = bicg_shifted_solve_dev(rank == 0 ? NULL : (bicg_matrix *)handle, 0, x, r, s, 2, 0, &st);  /* one rank: null handle */
    printf("rank %d:", rank);
    for (int i = 0; i < 7; ++i) printf(" %d", v[i]);
    printf("\n");
    bicg_shm_shutdown();
    return 0;
}
"""


def test_argument_check_is_collective(B, tmp_path):
    """A bad argument on one rank, or ranks that disagree on sigma_len, seed or method, make every rank return -1 before any
    device work, so no rank is left waiting for the others inside the solve."""
    src = tmp_path / "collective.c"
    src.write_text(_COLLECTIVE_C)
    exe = tmp_path / "collective"
    libdir = os.path.join(ROOT, "mpi-bicgstab_b200")
    subprocess.run(["gcc", "-O1", "-I" + os.path.join(ROOT, "include"), str(src), "-L" + libdir, "-lbicgstab_b200",
                    "-Wl,-rpath," + libdir, "-o", str(exe)], check=True)
    p = subprocess.run([os.path.join(ROOT, "tools", "bicgrun"), "-np", "3", str(exe)], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(l for l in p.stdout.splitlines() if l.startswith("rank ")) == [f"rank {r}: " + " ".join(["-1"] * 7) for r in range(3)]


# ---- the Python wrappers reject bad vectors before the library sees them --------------------------------------------------
@pytest.fixture
def dm(B):
    """A DeviceMatrix whose handle is never used: every call below must fail in Python."""
    blk = B.gen_block("stencil15", 4, 14.0)
    d = B.DeviceMatrix.__new__(B.DeviceMatrix)
    d.blk, d.h = blk, None
    yield d
    d.h = None


def _reject(fn, exc, text):
    with pytest.raises(exc, match=text):
        fn()


def test_shifted_solve_rejects_bad_tensors(B, dm):
    import torch
    n, L = dm.blk.n_loc, 3
    sigma = np.array([0.1, 0.2, 0.3])
    good_x, good_r = torch.zeros(L, n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    f = lambda x, r, s=sigma: dm.shifted_solve("shifted_lopbicgstab", x, r, s, 0)
    _reject(lambda: f(np.zeros((L, n)), good_r), TypeError, "cannot be mixed")                  # numpy / tensor mix
    _reject(lambda: f(good_x, np.zeros(n)), TypeError, "cannot be mixed")
    _reject(lambda: f(good_x.float(), good_r), TypeError, "float64")                            # wrong dtype
    _reject(lambda: f(good_x, good_r.to(torch.int64)), TypeError, "float64")
    _reject(lambda: f(torch.zeros(n, L, dtype=torch.float64).t(), good_r), ValueError, "contiguous")   # non-contiguous
    _reject(lambda: f(good_x, torch.zeros(2 * n, dtype=torch.float64)[::2]), ValueError, "contiguous")
    _reject(lambda: f(torch.zeros(L + 1, n, dtype=torch.float64), good_r), ValueError, "shape")  # sigma_len mismatch
    _reject(lambda: f(torch.zeros(L * n, dtype=torch.float64), good_r), ValueError, "shape")     # flat x_set
    _reject(lambda: f(good_x, torch.zeros(n + 1, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(good_x, good_r, torch.tensor([0.1, 0.2])), ValueError, "shape")           # sigma tensor of the wrong length
    _reject(lambda: f(good_x, good_r), TypeError, "CUDA")                                        # CPU tensors
    if torch.cuda.is_available():
        _reject(lambda: f(good_x.cuda(), good_r), TypeError, "CUDA")                             # CPU / CUDA mix


def test_solve_rejects_bad_tensors(B, dm):
    import torch
    n = dm.blk.n_loc
    x, r = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    f = lambda a, b: dm.solve("bicgstab", a, b)
    _reject(lambda: f(np.zeros(n), r), TypeError, "cannot be mixed")
    _reject(lambda: f(x, np.zeros(n)), TypeError, "cannot be mixed")
    _reject(lambda: f(x.float(), r), TypeError, "float64")
    _reject(lambda: f(x, torch.zeros(2 * n, dtype=torch.float64)[1::2]), ValueError, "contiguous")
    _reject(lambda: f(x, torch.zeros(n - 1, dtype=torch.float64)), ValueError, "shape")
    _reject(lambda: f(x.reshape(1, n), r), ValueError, "shape")
    _reject(lambda: f(x, r), TypeError, "CUDA")
    if torch.cuda.is_available():
        _reject(lambda: f(x, r.cuda()), TypeError, "CUDA")
