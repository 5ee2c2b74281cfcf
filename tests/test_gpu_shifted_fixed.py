"""GPU parity of shifted_lopbicg (-m gpu), the fixed-seed solver of shifted_switching_solver.h:11, through the C ABI against the
oracle restatement (oracle/shifted_fixed_oracle.c), which is pinned bitwise to the reference's own compiled function
(tests/test_oracle_golden_shifted_fixed.py).

Tolerances come from the oracle's own spread over summation orders (its P = 1, 2, 4, 8 emulations), not from a GPU run:
  * seed residual history, iterations 1..10: <= 1e-10 relative.  It is not compared later: once the seed has converged and keeps
    iterating, its recursive residual falls far below rounding (2.6e-39 on sh_convdiff_g40_L6_switch), where two summation
    orders do not agree relatively;
  * return value and every shift's stop iteration: within 2 of the range the oracle's P = 1, 2, 4, 8 runs span; on the
    250 k-row 64-shift cases, whose counts are chaotic like plain BiCGStab's on that matrix, within max(2, 10 %) of it;
  * every shift's true residual ||(A + sigma_j I) x_j - b|| <= max(10 x the oracle's, 1e-10 ||b||)."""
import ctypes as C
import re

import numpy as np
import pytest
import shifted_fixed_oracle as OF

from helpers import global_csr
from shifted_fixed_cases import FIXED_CASES, FIXED_LARGE_CASES, fixed_problem

pytestmark = pytest.mark.gpu
MAX_ITER = 1000
SPREAD_P = (1, 2, 4, 8)


def _oracles(n, ptr, col, val, b, sigma, seed, tol):
    return [OF.shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, P=P, tol=tol, max_iter=MAX_ITER) for P in SPREAD_P]


def _window(values, rel):
    lo, hi = min(values), max(values)
    return lo - max(2, int(rel * lo)), hi + max(2, int(rel * hi))


def _check(B, O, n, ptr, col, val, sigma, b, seed, ret, x, r, hist, st, refs, what, rel=0.0):
    """refs: the oracle at P = 1, 2, 4, 8 (refs[0] is P = 1).  Returns the GPU's stop iterations."""
    ref = refs[0]
    assert ret == st["iters"] and hist.size == ret + 1 and hist[0] == 1.0, what
    m = min(10, ret, ref["ret"])
    got, want = np.sqrt(hist[1:m + 1]), np.sqrt(ref["hist"][1:m + 1])
    assert np.all(np.abs(got - want) <= 1e-10 * want + 1e-15), (what, np.abs(got - want) / want)
    assert max(f["ret"] for f in refs) < MAX_ITER and st["converged"] == 1, what      # every case converges
    lo, hi = _window([f["ret"] for f in refs], rel)
    assert lo <= ret <= hi, (what, ret, [f["ret"] for f in refs])
    end_seed, stop = B.last_shift_info(sigma.size)
    assert end_seed == seed, what
    for j in range(sigma.size):
        lo, hi = _window([int(f["stop_iter"][j]) for f in refs], rel)
        assert lo <= stop[j] <= hi and 1 <= stop[j] <= ret, (what, j, stop[j], [int(f["stop_iter"][j]) for f in refs])
    nb = np.linalg.norm(b)
    for j in range(sigma.size):
        res = np.linalg.norm(O.spmv(n, ptr, col, val, x[j]) + sigma[j] * x[j] - b)
        res_ref = np.linalg.norm(O.spmv(n, ptr, col, val, ref["x"][j]) + sigma[j] * ref["x"][j] - b)
        assert res <= max(10 * res_ref, 1e-10 * nb), (what, j, res / nb, res_ref / nb)
    # the returned r is the seed system's recursive residual
    assert abs(np.dot(r, r) / np.dot(b, b) - hist[ret]) <= 1e-8 * max(hist[ret], 1e-300), what
    return stop


def _solve(B, blk, n, sigma, b, seed):
    x = np.zeros((sigma.size, n)); r = b.copy()
    ret = B.shifted_lopbicg(blk, x, r, sigma, seed)
    return ret, x, r, B.last_history(), B.last_stats()


@pytest.mark.parametrize("case", FIXED_CASES, ids=[c[0] for c in FIXED_CASES])
def test_fixed_matches_oracle(B, O, case):
    B.set_options(quiet=1, cache=1, shift_tol=case[7], shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    refs = _oracles(n, ptr, col, val, b, sigma, seed, tol)
    ret, x, r, hist, st = _solve(B, blk, n, sigma, b, seed)
    stop = _check(B, O, n, ptr, col, val, sigma, b, seed, ret, x, r, hist, st, refs, case[0])
    if case[0].endswith("_switch"):
        # the seed converges first (where the switching solver would switch) and keeps iterating for the other shifts
        assert refs[0]["stop_iter"][seed] < refs[0]["ret"]
        assert stop[seed] < ret, (stop, ret)
    if sigma.size == 1 or case[0].startswith("fx_"):
        assert np.abs(x[seed] - 1.0).max() < 1e-8


@pytest.mark.parametrize("case", FIXED_LARGE_CASES, ids=[c[0] for c in FIXED_LARGE_CASES])
def test_fixed_many_shifts(B, O, case):
    """main_shifted.c's 512 shifts on a small matrix (the whole coefficient table of the fused pass in shared memory), and 64
    shifts on the 250 k-row T' matrix with seed 0 and with seed 63, the largest shift: the oracle's fixed seed 63 needs 180
    iterations to 1e-10 at P = 1 where the switching solver needs 164.  The 64-shift counts are chaotic in the summation order
    of the dots, so they get the max(2, 10 %) window around the oracle's spread."""
    B.set_options(quiet=1, shift_tol=case[7], shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    refs = _oracles(n, ptr, col, val, b, sigma, seed, tol)
    ret, x, r, hist, st = _solve(B, blk, n, sigma, b, seed)
    B.set_options(shift_tol=1e-12)
    _check(B, O, n, ptr, col, val, sigma, b, seed, ret, x, r, hist, st, refs, case[0], rel=0.1 if case[2] == 63 else 0.0)


@pytest.mark.parametrize("case", FIXED_CASES[:3], ids=[c[0] for c in FIXED_CASES[:3]])
def test_fixed_is_the_switching_solve_until_the_switch(B, O, case):
    """On the same cached matrix the GPU's fixed and switching solves share their bits until the seed switch; without a switch
    (sh_stencil15_g12_L5) they are the same solve and the fixed one returns one less."""
    B.set_options(quiet=1, cache=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    ret, x, r, hist, st = _solve(B, blk, n, sigma, b, seed)
    _, stop = B.last_shift_info(sigma.size)
    xs = np.zeros((sigma.size, n)); rs = b.copy()
    ret_sw = B.shifted_lopbicg_switching(blk, xs, rs, sigma, seed)
    hist_sw = B.last_history()
    seed_sw, stop_sw = B.last_shift_info(sigma.size)
    k_s = int(stop[seed])
    if seed_sw == seed:
        assert ret_sw == ret + 1 and np.array_equal(hist, hist_sw) and np.array_equal(x, xs) and np.array_equal(r, rs)
        assert np.array_equal(stop, stop_sw)
    else:
        assert k_s == stop_sw[seed] and np.array_equal(hist[:k_s + 1], hist_sw[:k_s + 1])
        for j in range(sigma.size):
            if j != seed and 0 < stop[j] <= k_s:
                assert stop_sw[j] == stop[j] and np.array_equal(x[j], xs[j]), j


def test_fixed_stdout_contract(B, O, capfd):
    """shifted_switching_solver.c:234-248 with DISPLAY_RESULT off: only `Total time` and `Avg time/iter` (= total / k)."""
    case = FIXED_CASES[1]                                                   # a switching case: no switch lines either
    B.set_options(quiet=0, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    x = np.zeros((sigma.size, n)); r = b.copy()
    ret = B.shifted_lopbicg(blk, x, r, sigma, seed)
    B.lib.bicg_synchronize()
    C.CDLL(None).fflush(None)
    out = capfd.readouterr().out
    B.set_options(quiet=1)
    total = float(re.search(r"^Total time   : (\S+) \[sec\.\] \n", out, flags=re.M).group(1))
    avg = float(re.search(r"^Avg time/iter: (\S+) \[sec\.\] \n", out, flags=re.M).group(1))
    assert abs(avg - total / ret) <= 1e-6 * total / ret, (avg, total, ret)
    assert "Total iter" not in out and "Final r" not in out and "seed: " not in out and "remain: " not in out and "sigma[" not in out
    assert len([l for l in out.splitlines() if l.strip()]) == 2, out


def test_fixed_solve_ex_and_argument_checks(B, O):
    """bicg_shifted_solve_ex with BICG_SHIFTED_LOPBICG (3) on a resident matrix is the solve of shifted_lopbicg; bad arguments
    give -1."""
    B.set_options(quiet=1, cache=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    case = FIXED_CASES[1]
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    refs = _oracles(n, ptr, col, val, b, sigma, seed, tol)
    dm = B.DeviceMatrix(blk)
    x = np.zeros((sigma.size, n)); r = b.copy()
    ret, st = dm.shifted_solve("shifted_lopbicg", x, r, sigma, seed)
    assert st["kernel_launches"] > 0 and st["loop_ms"] > 0
    _check(B, O, n, ptr, col, val, sigma, b, seed, ret, x, r, B.last_history(), st, refs, "solve_ex")
    ret_entry = _solve(B, blk, n, sigma, b, seed)[0]
    assert ret == ret_entry
    x = np.zeros((sigma.size, n)); r = b.copy(); sg = np.ascontiguousarray(sigma)
    for method, L, sd in ((3, 0, 0), (3, sigma.size, sigma.size), (3, sigma.size, -1), (7, sigma.size, 0)):
        assert B.lib.bicg_shifted_solve_ex(dm.h, method, x.ctypes.data, r.ctypes.data, sg.ctypes.data, L, sd, None) == -1
    for L, sd in ((0, 0), (sigma.size, sigma.size), (sigma.size, -1)):
        assert B.lib.shifted_lopbicg(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), x.ctypes.data, r.ctypes.data,
                                     sg.ctypes.data, L, sd) == -1
    dm.destroy()
