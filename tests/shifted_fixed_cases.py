"""Test inputs of shifted_lopbicg, the fixed-seed solver of shifted_switching_solver.h:11: the SHIFTED_LOP_CASES (the switching
solver's SHIFTED_CASES plus test_shifted.c's set-up), a seed-only system and other seeds on test_shifted.c's shifts, and the
many-shift set-ups of main_shifted.c (512 shifts on a small matrix; 64 shifts on the 250 k-row T' matrix, whose seed 63 is the
largest shift: there the fixed seed needs more iterations than the switching solver)."""
import os

from shifted_lop_cases import GOLDEN_DIR, SHIFTED_LOP_CASES, shifted_lop_problem

# (name, kind, g, p0, number of shifts, shift scale, seed index, tol); scale None marks test_shifted.c's sigma_i = 0.01 i + 0.01
FIXED_CASES = [c + (1e-12,) for c in SHIFTED_LOP_CASES] + [
    ("fx_stencil15_g12_L1", "stencil15", 12, 14.0, 1, None, 0, 1e-12),
    ("fx_stencil15_g12_L5_seed2", "stencil15", 12, 14.0, 5, None, 2, 1e-12),
    ("fx_stencil15_g12_L5_seed4", "stencil15", 12, 14.0, 5, None, 4, 1e-12),
]
# golden data keeps only a digest of x and r for these, so that the file stays under 1 MB
FIXED_LARGE_CASES = [
    ("fx_stencil15_g12_L512", "stencil15", 12, 14.0, 512, 0.01 / 512, 0, 1e-12),
    ("fx_stencil15_g12_L512_seed511", "stencil15", 12, 14.0, 512, 0.01 / 512, 511, 1e-12),
    ("fx_stencil15_g63_L64", "stencil15", 63, 14.0, 64, 0.5 / 64, 0, 1e-10),
    ("fx_stencil15_g63_L64_seed63", "stencil15", 63, 14.0, 64, 0.5 / 64, 63, 1e-10),
]
GOLDEN_FIXED = os.path.join(GOLDEN_DIR, "ref_shifted_fixed.npz")


def fixed_problem(O, n, ptr, col, val, case):
    """sigma, b = (A + sigma[seed] I) 1, seed and tol of a FIXED_CASES / FIXED_LARGE_CASES entry."""
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case[:7])
    return sigma, b, seed, case[7]
