"""CPU: shifted_lopbicg (shifted_switching_solver.h:11) in the C ABI -- it is exported and declared with method 3 of
bicg_shifted_solve_ex, a program that declares the three prototypes of shifted_switching_solver.h and calls shifted_lopbicg links
against the library, and the reference's main_seed_diff.c with its commented-out shifted_lopbicg call swapped in links too (where a
checkout of the reference exists; compiled from a temporary copy, nothing of it is kept)."""
import os
import re
import subprocess

import pytest

from test_abi import REF_SRC, ROOT, _exported

PROTOTYPES = """
typedef struct CSR_Matrix CSR_Matrix;
typedef struct INFO_Matrix INFO_Matrix;
int shifted_lopbicg(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc, double *sigma, int sigma_len, int seed);
int shifted_lopbicg_switching(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc, double *sigma, int sigma_len, int seed);
int shifted_lopbicg_switching_noovlp(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc, double *sigma, int sigma_len, int seed);
"""


def _link(B, src, exe, extra=()):
    libdir = os.path.dirname(B.LIB_PATH)
    subprocess.run(["gcc", "-O2", "-w", *extra, str(src), "-L" + libdir, "-lbicgstab_b200", "-Wl,-rpath," + libdir, "-lm", "-o", str(exe)],
                   check=True)


def test_shifted_lopbicg_is_exported_and_declared(B):
    assert "shifted_lopbicg" in _exported(B)
    hdr = open(os.path.join(ROOT, "include", "bicgstab_b200.h")).read()
    assert re.search(r"\bint shifted_lopbicg\(CSR_Matrix \*A_loc_diag,", hdr)
    assert "BICG_SHIFTED_LOPBICG = 3" in hdr
    assert B.SHIFTED_SOLVE_EX == dict(B.SHIFTED_METHODS, shifted_lopbicg=3)
    assert "shifted_lopbicg" not in B.SHIFTED_METHODS


def test_program_calling_shifted_lopbicg_links(B, tmp_path):
    src = tmp_path / "fixed.c"
    src.write_text(PROTOTYPES + """
int main(int argc, char **argv)
{
    (void)argv;
    if (argc > 8) return shifted_lopbicg(0, 0, 0, 0, 0, 0, 0, 0) + shifted_lopbicg_switching(0, 0, 0, 0, 0, 0, 0, 0) +
                         shifted_lopbicg_switching_noovlp(0, 0, 0, 0, 0, 0, 0, 0);
    return 0;
}
""")
    exe = tmp_path / "fixed"
    _link(B, src, exe)
    assert subprocess.run([str(exe)]).returncode == 0
    undef = subprocess.run(["nm", "-u", str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert "shifted_lopbicg" in undef


def test_main_seed_diff_with_the_fixed_seed_call_links(B, tmp_path):
    """main_seed_diff.c:133-134 with the two comment markers swapped, the edit a user makes to compare a fixed seed with a
    switched one."""
    driver = os.path.join(REF_SRC, "main_seed_diff.c")
    if not os.path.isabs(driver) or not os.path.exists(driver):
        pytest.skip("no checkout of the reference")
    text = open(driver).read()
    swapped, n1 = re.subn(r"//(\s*total_iter = shifted_lopbicg\()", r"\1", text)
    swapped, n2 = re.subn(r"^(\s*)(total_iter = shifted_lopbicg_switching\()", r"\1//\2", swapped, flags=re.M)
    assert n1 == 1 and n2 == 1
    src = tmp_path / "main_seed_diff_fixed.c"
    src.write_text(swapped)
    exe = tmp_path / "main_seed_diff_fixed"
    _link(B, src, exe, ["-I" + os.path.join(ROOT, "include", "compat"), "-I" + REF_SRC])
    undef = subprocess.run(["nm", "-u", str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert "shifted_lopbicg" in undef and "shifted_lopbicg_switching" not in undef


def test_shifted_lopbicg_fails_loudly_without_gpu(B):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    code = ("import sys; sys.path.insert(0, %r); import numpy as np; import mpi_bicgstab_b200 as B; "
            "blk = B.gen_block('laplace5', 8); x = np.zeros((3, blk.n)); b = np.ones(blk.n); "
            "B.shifted_lopbicg(blk, x, b, np.array([0.1, 0.2, 0.3]), 0); print('RETURNED')" % ROOT)
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True)
    assert p.returncode == 1 and "RETURNED" not in p.stdout and "no usable CUDA device" in p.stderr
