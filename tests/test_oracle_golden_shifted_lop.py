"""CPU: the oracle's restatement of the LOP family of shifted_solver.h (shifted_lopbicgstab, shifted_pipe_lopbicgstab) is
bit-identical to what the reference's own compiled functions produced (tests/golden/ref_shifted_lop_<function>.npz, generator
tests/golden/make_golden_shifted_lop.py): return value, every x_j, the seed residual r and the residual history.  The golden data
also pins that the reference's twins (_v2, _nooverlap) compute exactly what their first function computes, which is why the
library maps each twin to the same solve."""
import numpy as np
import pytest
import shifted_lop_oracle as OL

from helpers import X0_GOLDEN, X0_SHIFTED_MAX_ITER, X0_SHIFTED_TOL, global_csr, x0_shifted_problem
from shifted_lop_cases import SHIFTED_LOP_CASES, SHIFTED_LOP_VARIANTS, golden_path, shifted_lop_problem

LOP = ["shifted_lopbicgstab", "shifted_lopbicgstab_v2", "shifted_lopbicgstab_nooverlap"]
PIPE = ["shifted_pipe_lopbicgstab", "shifted_pipe_lopbicgstab_nooverlap"]


def _gold(variant, name):
    g = np.load(golden_path(variant))
    return {k: g[f"{name}|{k}"] for k in ("ret", "x", "r", "res")}


@pytest.mark.parametrize("pipe", [False, True], ids=["lop", "pipe_lop"])
@pytest.mark.parametrize("case", SHIFTED_LOP_CASES, ids=[c[0] for c in SHIFTED_LOP_CASES])
def test_oracle_matches_reference_bitwise(B, O, case, pipe):
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    got = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, tol=1e-12, max_iter=1000)
    want = _gold(PIPE[0] if pipe else LOP[0], case[0])
    assert got["ret"] == int(want["ret"])
    assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["r"], want["r"])
    assert np.array_equal(np.sqrt(got["hist"][1:]), want["res"])        # the reference prints every iteration (OUT_ITER = 1)


@pytest.mark.parametrize("case", SHIFTED_LOP_CASES, ids=[c[0] for c in SHIFTED_LOP_CASES])
def test_reference_twins_are_bit_identical(case):
    for family in (LOP, PIPE):
        first = _gold(family[0], case[0])
        for twin in family[1:]:
            other = _gold(twin, case[0])
            for k in ("ret", "x", "r", "res"):
                assert np.array_equal(first[k], other[k]), (twin, k)


@pytest.mark.parametrize("case", SHIFTED_LOP_CASES, ids=[c[0] for c in SHIFTED_LOP_CASES])
def test_lop_solves_every_shifted_system(B, O, case):
    """LOP keeps its accuracy: every x_j the reference returns solves (A + sigma_j I) x_j = b to 1e-10 |b|.  (PIPE-LOP does not
    always: it stops at MAX_ITER on sh_convdiff_g40_L6_switch and reaches about 5e-9 on sh_stencil15_g12_L4_switch.)"""
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    x = _gold(LOP[0], case[0])["x"]
    for j in range(sigma.size):
        res = O.spmv(n, ptr, col, val, x[j]) + sigma[j] * x[j] - b
        assert np.linalg.norm(res) <= 1e-10 * np.linalg.norm(b), (j, np.linalg.norm(res) / np.linalg.norm(b))


@pytest.mark.parametrize("pipe", [False, True], ids=["lop", "pipe_lop"])
def test_oracle_from_nonzero_x0_matches_reference_bitwise(B, O, pipe):
    """From a nonzero x_set (tests/golden/ref_x0.npz): the reference's return value, every x_j, r and printed residual."""
    gold = np.load(X0_GOLDEN)
    n, ptr, col, val, b, sigma, seed, x0 = x0_shifted_problem(B, O, gold)
    got = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, tol=X0_SHIFTED_TOL, max_iter=X0_SHIFTED_MAX_ITER, x0=x0)
    want = {k: gold[f"shifted|{PIPE[0] if pipe else LOP[0]}|{k}"] for k in ("ret", "res", "x", "r")}
    assert got["ret"] == want["ret"]
    assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["r"], want["r"])
    assert np.array_equal(np.sqrt(got["hist"][1:]), want["res"])


def test_golden_covers_every_reference_function():
    for v in SHIFTED_LOP_VARIANTS:
        g = np.load(golden_path(v))
        assert all(f"{c[0]}|ret" in g for c in SHIFTED_LOP_CASES), v
