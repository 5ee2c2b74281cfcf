"""GPU: the fused multi-shift residual check (csrc/shift_check.cu).

* bicg_shift_residuals against an exact host evaluation (long double components of A x_j + sigma_j x_j - b, math.fsum norms), for
  L in {1, 5, 64, 512} (batch remainders), on stencil15, convdiff, laplace5 and random k = 32 matrices, n = 17 and n not a multiple
  of 16, host and device vectors, random x_j (relative error <= 1e-13) and the converged x_j of a solve, whose tiny residual is held
  to 1e-13 (|| |A| |x_j| || + |sigma_j| ||x_j|| + ||b||) / ||b||; L = 513, 1100 and 4000 take several launches.
* BICG_SHIFT_ERROR=1 for each of the four shifted methods: the reference's printout (shifted_switching_solver.c:572, 593-594), its
  values equal to bicg_last_shift_error to %e precision and to the exact evaluation of the returned x_j, and x_set, r, the return
  value, the statistics and the history identical to a run with the option off, whose stdout carries no error block; a solve
  after the report is bit-identical to one before it.  Also after solves with 4000 shifts.
* test_shifted.c -DDISPLAY_ERROR linked against the library (oracle/_ref/ref_test_shifted_error_b200) on the golden .mtx."""
import ctypes as C
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import SHIFTED_CASES, global_csr
from shifted_lop_cases import SHIFTED_LOP_CASES, mtx_path, shifted_lop_problem

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ITER = 1000
MATRICES = [("stencil15", 12, 14.0), ("convdiff", 40, 1.5), ("laplace5", 37, 0.0), ("random", 3001, 32), ("random", 17, 5)]
METHODS = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]


def exact_errors(ptr, col, val, x_set, b, sigma):
    """(relative errors, bound scale) of every shift: components in long double, norms with math.fsum.  scale[j] =
    (|| |A| |x_j| || + |sigma_j| ||x_j|| + ||b||) / ||b||, the size of what the rounding of one component can reach."""
    ptr = np.asarray(ptr, dtype=np.int64)
    rows = np.repeat(np.arange(ptr.size - 1), np.diff(ptr))
    vl = np.asarray(val, dtype=np.longdouble)
    bl = np.asarray(b, dtype=np.longdouble)
    nb = math.sqrt(math.fsum(float(v) * float(v) for v in b))
    err, scale = [], []
    for j in range(len(sigma)):
        xl = np.asarray(x_set[j], dtype=np.longdouble)
        ax = np.zeros(b.size, dtype=np.longdouble)
        np.add.at(ax, rows, vl * xl[col])
        d = ax + np.longdouble(sigma[j]) * xl - bl
        err.append(math.sqrt(math.fsum((float(v) for v in d * d))) / nb)
        aax = np.zeros(b.size)
        np.add.at(aax, rows, np.abs(val) * np.abs(x_set[j][col]))
        scale.append((np.linalg.norm(aax) + abs(sigma[j]) * np.linalg.norm(x_set[j]) + nb) / nb)
    return np.array(err), np.array(scale)


def _residuals(B, dm, x, b, sigma, device):
    if not device:
        return dm.shift_residuals(x, b, sigma)
    import torch
    return dm.shift_residuals(torch.from_numpy(x).cuda(), torch.from_numpy(b).cuda(), sigma)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("L", [1, 5, 64, 512])
@pytest.mark.parametrize("mat", MATRICES, ids=[f"{k}{g}" for k, g, _ in MATRICES])
def test_shift_residuals_random_x(B, mat, L, device):
    blk, n, ptr, col, val = global_csr(B, *mat)
    rng = np.random.default_rng(L * 1000 + n)
    x = rng.standard_normal((L, n))
    b = rng.standard_normal(n)
    sigma = rng.uniform(-0.5, 0.5, L)
    dm = B.DeviceMatrix(blk)
    got = _residuals(B, dm, x, b, sigma, device)
    dm.destroy()
    want, _ = exact_errors(ptr, col, val, x, b, sigma)
    assert got.shape == (L,)
    assert np.all(np.abs(got - want) <= 1e-13 * want), (mat, L, np.abs(got - want) / want)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("case", SHIFTED_CASES[:1] + SHIFTED_CASES[3:], ids=[c[0] for c in SHIFTED_CASES[:1] + SHIFTED_CASES[3:]])
def test_shift_residuals_converged_x(B, O, case, device):
    B.set_options(quiet=1, shift_error=0, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    dm = B.DeviceMatrix(blk)
    x = np.zeros((sigma.size, n)); r = b.copy()
    dm.shifted_solve("shifted_lopbicgstab", x, r, sigma, seed)
    got = _residuals(B, dm, x, b, sigma, device)
    dm.destroy()
    want, scale = exact_errors(ptr, col, val, x, b, sigma)
    assert np.all(np.abs(got - want) <= 1e-13 * scale), (case[0], got, want)
    assert np.all(want < 1e-9)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("L", [513, 1100, 4000])
def test_shift_residuals_many_shifts(B, L, device):
    """More shifts than one launch takes (512): a second launch with one shift, three launches, and L = 4000, whose per-warp
    partials would not fit a CTA's shared memory in one launch."""
    blk, n, ptr, col, val = global_csr(B, "random", 17, 5)
    rng = np.random.default_rng(L)
    x = rng.standard_normal((L, n)); b = rng.standard_normal(n); sigma = rng.uniform(-0.5, 0.5, L)
    dm = B.DeviceMatrix(blk)
    got = _residuals(B, dm, x, b, sigma, device)
    dm.destroy()
    want, _ = exact_errors(ptr, col, val, x, b, sigma)
    assert got.shape == (L,) and np.all(np.abs(got - want) <= 1e-13 * want), (L, np.abs(got - want).max())


@pytest.mark.parametrize("method", ["shifted_lopbicg_switching", "shifted_lopbicgstab"])
def test_in_solver_report_many_shifts(B, O, method):
    """BICG_SHIFT_ERROR=1 after a solve with 4000 shifts, which the solvers take."""
    B.set_options(quiet=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, "random", 17, 5)
    L, seed = 4000, 0
    sigma = (np.arange(L) + 1) * (0.01 / L)
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[seed], np.ones(n), b)
    dm = B.DeviceMatrix(blk)
    B.set_options(shift_error=1)
    x = np.zeros((L, n)); r = b.copy()
    dm.shifted_solve(method, x, r, sigma, seed)
    B.set_options(shift_error=0)
    err = B.last_shift_error(L)
    dm.destroy()
    want, scale = exact_errors(ptr, col, val, x, b, sigma)
    assert err.size == L and np.all(np.abs(err - want) <= 1e-13 * scale), (method, np.abs(err - want).max())


def test_shift_residuals_long_rows(B):
    """Rows of 2000 entries, longer than any SpMV stage: the thread-per-row walk needs no chunking."""
    blk, n, ptr, col, val = global_csr(B, "random", 2111, 2000)
    rng = np.random.default_rng(7)
    L = 9
    x = rng.standard_normal((L, n)); b = rng.standard_normal(n); sigma = rng.uniform(0, 1, L)
    dm = B.DeviceMatrix(blk)
    got = dm.shift_residuals(x, b, sigma)
    dm.destroy()
    want, _ = exact_errors(ptr, col, val, x, b, sigma)
    assert np.all(np.abs(got - want) <= 1e-13 * want)


_ERR_LINE = re.compile(r"^([01]), (\S+), (\S+)$")


def _run(B, dm, method, sigma, b, seed, capfd, on):
    B.set_options(shift_error=1 if on else 0)
    x = np.zeros((sigma.size, b.size)); r = b.copy()
    ret, st = dm.shifted_solve(method, x, r, sigma, seed)
    B.lib.bicg_synchronize()
    C.CDLL(None).fflush(None)
    out = capfd.readouterr().out
    B.set_options(shift_error=0)
    return ret, st, x, r, out, B.last_shift_error(sigma.size), B.last_history()


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", [SHIFTED_LOP_CASES[0], SHIFTED_CASES[1], SHIFTED_LOP_CASES[-1], SHIFTED_CASES[3]],
                         ids=lambda c: c[0])
def test_in_solver_report(B, O, capfd, method, case):
    B.set_options(quiet=0, cache=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    dm = B.DeviceMatrix(blk)
    capfd.readouterr()
    off = _run(B, dm, method, sigma, b, seed, capfd, False)
    on = _run(B, dm, method, sigma, b, seed, capfd, True)
    final_seed = B.last_shift_info(sigma.size)[0] if method in ("shifted_lopbicg_switching", "shifted_lopbicg") else seed
    again = _run(B, dm, method, sigma, b, seed, capfd, False)
    dm.destroy()
    B.set_options(quiet=1)
    # the option changes nothing the solve returns (the check runs after the solve's statistics are taken, so the stats are
    # compared for what the caller receives), and it leaves the handle as a solve left it: the next solve is bit-identical
    for other in (on, again):
        assert other[0] == off[0] and other[1]["kernel_launches"] == off[1]["kernel_launches"]
        assert other[1]["iters"] == off[1]["iters"] and other[1]["converged"] == off[1]["converged"]
        assert np.array_equal(other[2], off[2], equal_nan=True) and np.array_equal(other[3], off[3], equal_nan=True)
        assert np.array_equal(other[6], off[6], equal_nan=True)
    assert "relative error" not in again[4] and again[5].size == 0
    # off: no error block, nothing kept
    assert "relative error" not in off[4] and off[5].size == 0
    mask = lambda s: re.sub(r"(Total time   :|Avg time/iter:) \S+", r"\1", s)
    head, sep, block = on[4].partition("seed(0:seed, 1:shift), sigma, relative error\n")
    assert sep and mask(head) == mask(off[4])                     # the solver's own lines come first, unchanged
    err = on[5]
    assert err.size == sigma.size
    shown = [i for i in range(sigma.size) if i == final_seed or i % 10 == 0]
    lines = block.splitlines()
    assert len(lines) == len(shown), (block, shown)
    for i, line in zip(shown, lines):
        m = _ERR_LINE.match(line)
        assert m and m.group(1) == ("0" if i == final_seed else "1") and m.group(2) == "%e" % sigma[i], (line, i)
        if np.isfinite(err[i]):
            assert m.group(3) == "%e" % err[i], (line, err[i])
        else:
            assert "nan" in m.group(3) or "inf" in m.group(3), line
    want, scale = exact_errors(ptr, col, val, on[2], b, sigma)
    fin = np.isfinite(want)
    assert np.array_equal(fin, np.isfinite(err))
    assert np.all(np.abs(err[fin] - want[fin]) <= 1e-13 * scale[fin]), (method, case[0], err, want)
    if case is SHIFTED_CASES[1]:
        assert method not in ("shifted_lopbicg_switching",) or final_seed != seed      # the switch case does switch


def test_quiet_suppresses_the_printout(B, O, capfd):
    case = SHIFTED_LOP_CASES[0]
    B.set_options(quiet=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    dm = B.DeviceMatrix(blk)
    capfd.readouterr()
    ret, st, x, r, out, err, _ = _run(B, dm, "shifted_lopbicgstab", sigma, b, seed, capfd, True)
    dm.destroy()
    assert out == "" and err.size == sigma.size


def test_test_shifted_display_error_driver(tmp_path):
    """test_shifted.c built with -DDISPLAY_ERROR, linked against the library: its five relative errors on the golden .mtx within
    max(10 x what the reference's own build printed, 1e-10)."""
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_test_shifted_error_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_test_shifted_error_b200 not built")
    with open(os.path.join(ROOT, "tests", "golden", "ref_shift_error.json")) as f:
        gold = json.load(f)["lines"]
    p = subprocess.run([exe, mtx_path()], capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    rows = [(m.group(1) == "#seed", float(m.group(2)), float(m.group(3)))
            for m in re.finditer(r"^(#seed|sigma): (\S+), relative error: (\S+)$", p.stdout, re.M)]
    assert len(rows) == 5, p.stdout
    for (is_seed, sg, e), g in zip(rows, gold):
        assert is_seed == g["seed"] and sg == g["sigma"]
        assert e <= max(10 * g["relative_error"], 1e-10), (e, g)
