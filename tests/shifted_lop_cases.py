"""Test inputs of the LOP family of shifted_solver.h (shifted_solver.c:182-1085): the SHIFTED_CASES of helpers.py plus
test_shifted.c's own set-up (test_shifted.c:13-14, 95-111: 5 shifts, sigma_i = 0.01 i + 0.01, seed 0) on the T' family."""
import os

import numpy as np

from helpers import SHIFTED_CASES, shifted_problem

# (name, kind, g, p0, number of shifts, shift scale, seed index); scale None marks test_shifted.c's set-up
SHIFTED_LOP_CASES = SHIFTED_CASES + [("sh_test_shifted_stencil15_g12", "stencil15", 12, 14.0, 5, None, 0)]
SHIFTED_LOP_VARIANTS = ["shifted_lopbicgstab", "shifted_lopbicgstab_v2", "shifted_lopbicgstab_nooverlap", "shifted_pipe_lopbicgstab",
                        "shifted_pipe_lopbicgstab_nooverlap"]
SHIFTED_LOP_MTX = ("convdiff", 16, 1.5)       # the small Matrix-Market file the unchanged test_shifted.c runs on
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_path(variant):
    """One file per reference function keeps every golden file under 1 MB."""
    return os.path.join(GOLDEN_DIR, f"ref_shifted_lop_{variant}.npz")


def mtx_path():
    kind, g, _ = SHIFTED_LOP_MTX
    return os.path.join(GOLDEN_DIR, f"test_shifted_{kind}{g}.mtx")


def shifted_lop_problem(O, n, ptr, col, val, case):
    """sigma, b = (A + sigma[seed] I) 1 and seed of a SHIFTED_LOP_CASES entry."""
    _, _, _, _, L, scale, seed = case
    if scale is not None:
        sigma, b = shifted_problem(O, n, ptr, col, val, L, scale, seed)
        return sigma, b, seed
    sigma = np.arange(L) * 0.01 + 0.01
    b = O.spmv(n, ptr, col, val, np.ones(n))
    O.daxpy(sigma[seed], np.ones(n), b)
    return sigma, b, seed
