"""CPU: the shifted-solution check in the C ABI -- bicg_shift_residuals / bicg_last_shift_error are declared and exported, the
SHIFT_ERROR option exists, the query refuses to run without a GPU, and the MPI_Allreduce of include/compat/mpi.h (what
test_shifted.c's DISPLAY_ERROR block calls) gives every rank the rank-ordered sum, so that driver links against the library."""
import ctypes as C
import os
import struct
import subprocess

import pytest

from test_abi import REF_SRC, ROOT, _exported

_ALLREDUCE_C = r"""
#include <stdio.h>
#include <mpi.h>
int main(int argc, char **argv)
{
    int rank, size;
    MPI_Init(&argc, &argv);
    MPI_Comm_rank(MPI_COMM_WORLD, &rank);
    MPI_Comm_size(MPI_COMM_WORLD, &size);
    double v[3] = {1.0 + rank, rank == 0 ? 1.0 : (rank == 1 ? 1e16 : -1e16), 0.1 * (rank + 1)}, out[3];
    MPI_Allreduce(v, out, 3, MPI_DOUBLE, MPI_SUM, MPI_COMM_WORLD);
    MPI_Allreduce(MPI_IN_PLACE, v, 3, MPI_DOUBLE, MPI_SUM, MPI_COMM_WORLD);
    printf("rank %d of %d:", rank, size);
    for (int i = 0; i < 3; ++i) printf(" %a %a", out[i], v[i]);
    printf("\n");
    MPI_Finalize();
    return 0;
}
"""

_BAD_OP_C = r"""
#include <stdio.h>
#include <mpi.h>
int main(int argc, char **argv)
{
    MPI_Init(&argc, &argv);
    double v = 1.0, w = 0.0;
    MPI_Allreduce(&v, &w, 1, %s, %s, MPI_COMM_WORLD);
    printf("RETURNED\n");
    MPI_Finalize();
    return 0;
}
"""


def _compile(tmp_path, name, source):
    src = tmp_path / f"{name}.c"
    src.write_text(source)
    exe = tmp_path / name
    libdir = os.path.join(ROOT, "mpi-bicgstab_b200")
    subprocess.run(["gcc", "-O1", "-I" + os.path.join(ROOT, "include", "compat"), str(src), "-L" + libdir, "-lbicgstab_b200",
                    "-Wl,-rpath," + libdir, "-o", str(exe)], check=True)
    return str(exe)


def test_query_is_declared_and_exported(B):
    with open(os.path.join(ROOT, "include", "bicgstab_b200.h")) as f:
        header = f.read()
    assert "int bicg_shift_residuals(bicg_matrix *m, const double *x_set, const double *b, const double *sigma, int sigma_len," in header
    assert "int bicg_last_shift_error(double *out, int cap);" in header
    exported = _exported(B)
    for sym in ("bicg_shift_residuals", "bicg_last_shift_error", "bicg_shim_MPI_Allreduce"):
        assert sym in exported, sym
    assert {"bicg_shift_residuals", "bicg_last_shift_error"} <= set(B.SYMBOLS)


def test_shift_error_option(B):
    assert B.lib.bicg_set_option(b"SHIFT_ERROR", b"1") == 0
    assert B.lib.bicg_set_option(b"BICG_SHIFT_ERROR", b"0") == 0
    B.set_options(shift_error=0)


def test_query_fails_loudly_without_gpu(B):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    # the handle is a zeroed buffer: the device check comes before anything reads it
    code = ("import sys, ctypes as C; sys.path.insert(0, %r); import numpy as np; import mpi_bicgstab_b200 as B; "
            "h = C.create_string_buffer(4096); x = np.zeros(8); b = np.ones(4); s = np.array([0.1, 0.2]); out = np.zeros(2); "
            "B.lib.bicg_shift_residuals(C.addressof(h), x.ctypes.data, b.ctypes.data, s.ctypes.data, 2, 0, "
            "out.ctypes.data_as(C.POINTER(C.c_double))); print('RETURNED')" % ROOT)
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


def test_query_rejects_bad_arguments(B):
    """Argument checks come before the device check, so they hold without a GPU too."""
    h = C.create_string_buffer(64)
    x = (C.c_double * 4)(); out = (C.c_double * 2)(); s = (C.c_double * 2)(0.1, 0.2)
    f = B.lib.bicg_shift_residuals
    assert f(C.addressof(h), x, x, s, 0, 0, out) == -1
    assert f(None, x, x, s, 2, 0, out) == -1
    assert f(C.addressof(h), None, x, s, 2, 0, out) == -1
    assert f(C.addressof(h), x, None, s, 2, 0, out) == -1
    assert f(C.addressof(h), x, x, None, 2, 0, out) == -1
    assert f(C.addressof(h), x, x, s, 2, 0, None) == -1


_COLLECTIVE_ARGS_C = r"""
#include <stdio.h>
#include "bicgstab_b200.h"
int bicg_shm_bootstrap(void); void bicg_shm_shutdown(void);
int main(void)
{
    bicg_shm_bootstrap();
    const int rank = bicg_comm_rank();
    static char handle[4096];                       /* never read: every call below fails its collective argument check */
    double x[8] = {0}, b[4] = {1, 1, 1, 1}, s[3] = {0.1, 0.2, 0.3}, out[3];
    int a = bicg_shift_residuals((bicg_matrix *)handle, x, b, s, 2, 0, rank == 1 ? NULL : out);   /* one rank: null out */
    int c = bicg_shift_residuals((bicg_matrix *)handle, x, b, s, rank == 2 ? 3 : 2, 0, out);      /* sigma_len differs */
    printf("rank %d: %d %d\n", rank, a, c);
    bicg_shm_shutdown();
    return 0;
}
"""


def test_query_argument_check_is_collective(B, tmp_path):
    """A bad argument on one rank, or ranks that disagree on sigma_len, make every rank return -1 (before any device work,
    so no rank is left waiting for the others in the residual pass)."""
    src = tmp_path / "collective.c"
    src.write_text(_COLLECTIVE_ARGS_C)
    exe = tmp_path / "collective"
    libdir = os.path.join(ROOT, "mpi-bicgstab_b200")
    subprocess.run(["gcc", "-O1", "-I" + os.path.join(ROOT, "include"), str(src), "-L" + libdir, "-lbicgstab_b200",
                    "-Wl,-rpath," + libdir, "-o", str(exe)], check=True)
    p = subprocess.run([os.path.join(ROOT, "tools", "bicgrun"), "-np", "3", str(exe)], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(l for l in p.stdout.splitlines() if l.startswith("rank ")) == [f"rank {r}: -1 -1" for r in range(3)]


def test_allreduce_three_ranks_rank_ordered(B, tmp_path):
    exe = _compile(tmp_path, "allreduce", _ALLREDUCE_C)
    p = subprocess.run([os.path.join(ROOT, "tools", "bicgrun"), "-np", "3", exe], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = sorted(l for l in p.stdout.splitlines() if l.startswith("rank "))
    assert len(lines) == 3, p.stdout
    contrib = [[1.0 + r, [1.0, 1e16, -1e16][r], 0.1 * (r + 1)] for r in range(3)]
    want = []
    for i in range(3):
        s = contrib[0][i]
        for r in (1, 2):
            s += contrib[r][i]
        want.append(s)
    for r, line in enumerate(lines):
        head, vals = line.split(":")
        assert head == f"rank {r} of 3"
        got = [float.fromhex(t) for t in vals.split()]
        assert got == [w for w in want for _ in (0, 1)], (line, want)     # MPI_IN_PLACE and not: the same bits
    # the rank-ordered sum is not the sum in any other order for this data
    assert struct.pack("<d", want[1]) != struct.pack("<d", contrib[0][1] + (contrib[1][1] + contrib[2][1]))


@pytest.mark.parametrize("dtype,op", [("MPI_DOUBLE", "2"), ("MPI_INT", "MPI_SUM")])
def test_allreduce_unsupported_type_or_op_exits(B, tmp_path, dtype, op):
    exe = _compile(tmp_path, "badop", _BAD_OP_C % (dtype, op))
    p = subprocess.run([exe], capture_output=True, text=True, timeout=60, env=dict(os.environ, WORLD_SIZE="1"))
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "MPI_Allreduce supports MPI_DOUBLE with MPI_SUM only" in p.stderr


def test_test_shifted_c_with_display_error_links(B, tmp_path):
    """With a checkout of the reference: its test_shifted.c built with -DDISPLAY_ERROR (which adds MPI_Allreduce) links against the
    library with include/compat/mpi.h."""
    src = os.path.join(REF_SRC, "test_shifted.c")
    if not os.path.exists(src):
        pytest.skip("no checkout of the reference")
    exe = tmp_path / "test_shifted_error"
    libdir = os.path.dirname(B.LIB_PATH)
    subprocess.run(["gcc", "-O2", "-w", "-DDISPLAY_ERROR", "-I" + os.path.join(ROOT, "include", "compat"), "-I" + REF_SRC, src,
                    "-L" + libdir, "-lbicgstab_b200", "-Wl,-rpath," + libdir, "-lm", "-o", str(exe)], check=True)
    assert os.path.exists(exe)
