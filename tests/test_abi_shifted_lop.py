"""CPU: the LOP family of shifted_solver.h in the C ABI -- the five reference entry points and bicg_shifted_solve_ex are exported
(shifted_bicgstab is not), a program using every external symbol of the reference's unchanged test_shifted.c links against the
library, and without a GPU the entry points refuse to run (message + exit(1), no CPU path)."""
import json
import os
import subprocess

import pytest

from test_abi import ROOT, _build_reference_driver, _exported

ENTRY_POINTS = ["shifted_lopbicgstab", "shifted_lopbicgstab_v2", "shifted_lopbicgstab_nooverlap", "shifted_pipe_lopbicgstab",
                "shifted_pipe_lopbicgstab_nooverlap"]


def test_entry_points_are_exported(B):
    exported = _exported(B)
    for sym in ENTRY_POINTS + ["bicg_shifted_solve_ex", "shifted_lopbicg_switching", "bicg_shifted_solve"]:
        assert sym in exported, sym
    assert "shifted_bicgstab" not in exported                       # shifted_solver.c:13-180 is not provided
    assert B.SHIFTED_METHODS == {"shifted_lopbicg_switching": 0, "shifted_lopbicgstab": 1, "shifted_pipe_lopbicgstab": 2}


def test_test_shifted_c_links_against_the_library(B, tmp_path):
    """A program that references every external symbol of the reference's unchanged test_shifted.c compiled against
    include/compat/mpi.h (golden list, tests/golden/make_golden_driver_test_shifted.py) links and runs against the library +
    libc / libm: the link fails if the library leaves one of them unresolved."""
    with open(os.path.join(ROOT, "tests", "golden", "ref_driver_test_shifted.json")) as f:
        syms = json.load(f)["test_shifted.c"]
    src = tmp_path / "uses.c"
    src.write_text("".join(f"extern void {s}(void);\n" for s in syms) +
                   "void (*volatile uses[])(void) = {" + ", ".join(syms) + "};\nint main(void) { return uses[0] == 0; }\n")
    exe = tmp_path / "uses"
    libdir = os.path.dirname(B.LIB_PATH)
    subprocess.run(["gcc", "-w", "-fno-builtin", str(src), "-L" + libdir, "-lbicgstab_b200", "-Wl,-rpath," + libdir, "-lm",
                    "-o", str(exe)], check=True)
    assert subprocess.run([str(exe)]).returncode == 0
    exported = _exported(B)
    for sym in ("shifted_pipe_lopbicgstab_nooverlap", "MPI_csr_spmv_ovlap", "MPI_csr_load_matrix_block", "my_daxpy", "my_dcopy"):
        assert sym in syms and sym in exported, sym
    _build_reference_driver(B, tmp_path, "test_shifted.c")          # with a checkout: the unchanged source links too


@pytest.mark.parametrize("entry", ["shifted_lopbicgstab", "shifted_pipe_lopbicgstab"])
def test_entry_points_fail_loudly_without_gpu(B, entry):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys; sys.path.insert(0, %r); import numpy as np; import mpi_bicgstab_b200 as B; "
            "blk = B.gen_block('laplace5', 8); x = np.zeros((3, blk.n)); b = np.ones(blk.n); "
            "B.%s(blk, x, b, np.array([0.1, 0.2, 0.3]), 0); print('RETURNED')" % (ROOT, entry))
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr


def test_unchanged_test_shifted_fails_loudly_without_gpu(B, tmp_path):
    """The unchanged test_shifted.c (built where a checkout of the reference exists) loads its matrix on the host, then its first
    device call must exit(1) with a message."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    exe = _build_reference_driver(B, tmp_path, "test_shifted.c")
    if not exe:
        pytest.skip("no checkout of the reference")
    mtx = tmp_path / "a.mtx"
    mtx.write_text("%%MatrixMarket matrix coordinate real general\n3 3 5\n1 1 4.0\n2 2 4.0\n3 3 4.0\n1 2 -1.0\n3 2 -1.0\n")
    p = subprocess.run([exe, str(mtx)], capture_output=True, text=True)
    assert p.returncode == 1 and "IO time" in p.stdout and "Total iter" not in p.stdout, (p.stdout, p.stderr)
    assert "no usable CUDA device" in p.stderr
