"""GPU parity of the LOP family of shifted_solver.h (-m gpu): shifted_lopbicgstab (LOP) and shifted_pipe_lopbicgstab (PIPE-LOP)
through the C ABI against the oracle restatement, which is pinned bitwise to the reference's own compiled sources
(tests/test_oracle_golden_shifted_lop.py).  Tolerances as for the switching solver and the un-shifted pipelined solvers: seed
residual history, iterations 1..10, <= 1e-10 relative; iteration count within max(2, 2 %), or MAX_ITER where the reference itself
stops there; every x_j solves its system to max(10 x the oracle's own true residual, 1e-10 |b|) where the reference converges
(PIPE-LOP loses attainable accuracy, so it is held to the reference's, not to EPS)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import shifted_lop_oracle as OL

from helpers import global_csr
from shifted_lop_cases import SHIFTED_LOP_CASES, SHIFTED_LOP_VARIANTS, golden_path, mtx_path, shifted_lop_problem

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ITER = 1000
ALGOS = [("lop", False), ("pipe_lop", True)]


def _entry(B, pipe):
    return B.shifted_pipe_lopbicgstab if pipe else B.shifted_lopbicgstab


def _true_res(O, n, ptr, col, val, sigma, x, b):
    return np.array([np.linalg.norm(O.spmv(n, ptr, col, val, x[j]) + sigma[j] * x[j] - b) for j in range(sigma.size)])


def _check(O, n, ptr, col, val, sigma, b, ret, x, r, hist, ref, max_iter=MAX_ITER, what="", spread=None, converged=None):
    """ref: the oracle at P = 1.  spread: per-iteration relative spread of the oracle's own histories over rank counts, which
    widens the 1e-10 history tolerance only where the recurrence itself amplifies rounding (see the non-converging case)."""
    m = min(10, ret, ref["ret"])
    got, want = np.sqrt(hist[1:m + 1]), np.sqrt(ref["hist"][1:m + 1])
    tol = 1e-10 if spread is None else np.maximum(1e-10, 10 * spread[:m])
    assert np.all(np.abs(got - want) <= tol * want + 1e-15), (what, np.abs(got - want) / want)
    if ref["ret"] >= max_iter:
        # the reference does not converge (PIPE-LOP, sh_convdiff_g40_L6_switch): its residual stagnates while the shifts'
        # |1/(zeta pi)| keeps growing.  The oracle stops at MAX_ITER for P = 1, 2 and breaks down with a NaN for P = 3, 4, 8:
        # which of the two happens depends on the summation order, so the GPU is only held to the same non-convergence.
        assert converged is not None and not converged, what
        fin = hist[np.isfinite(hist)]
        assert fin.min() <= 10 * np.nanmin(ref["hist"]), (what, fin.min(), np.nanmin(ref["hist"]))
        return
    assert abs(ret - ref["ret"]) <= max(2, int(0.02 * ref["ret"])), (what, ret, ref["ret"])
    res = _true_res(O, n, ptr, col, val, sigma, x, b)
    res_ref = _true_res(O, n, ptr, col, val, sigma, ref["x"], b)
    bound = np.maximum(10 * res_ref, 1e-10 * np.linalg.norm(b))
    assert np.all(res <= bound), (what, res / np.linalg.norm(b), res_ref / np.linalg.norm(b))
    # the returned r is the seed system's recursive residual
    assert abs(np.dot(r, r) / np.dot(b, b) - hist[ret]) <= 1e-8 * max(hist[ret], 1e-300), what


def _spread(O, n, ptr, col, val, b, sigma, seed, pipe, ref):
    """Largest relative deviation of the oracle's P = 2, 3, 4, 8 histories (iterations 1..10) from its P = 1 history."""
    h1 = np.sqrt(ref["hist"][1:11])
    out = np.zeros(h1.size)
    for P in (2, 3, 4, 8):
        h = np.sqrt(OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, P=P, tol=1e-12, max_iter=MAX_ITER)["hist"][1:11])
        k = min(h.size, h1.size)
        out[:k] = np.maximum(out[:k], np.abs(h[:k] - h1[:k]) / h1[:k])
    return out


@pytest.mark.parametrize("algo,pipe", ALGOS)
@pytest.mark.parametrize("case", SHIFTED_LOP_CASES, ids=[c[0] for c in SHIFTED_LOP_CASES])
def test_shifted_lop_matches_oracle(B, O, algo, pipe, case):
    B.set_options(quiet=1, cache=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    ref = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, tol=1e-12, max_iter=MAX_ITER)
    x = np.zeros((sigma.size, n))
    r = b.copy()
    ret = _entry(B, pipe)(blk, x, r, sigma, seed)
    hist = B.last_history()
    st = B.last_stats()
    assert hist.size == ret + 1 and st["iters"] == ret
    _check(O, n, ptr, col, val, sigma, b, ret, x, r, hist, ref, what=(case[0], algo),
           spread=_spread(O, n, ptr, col, val, b, sigma, seed, pipe, ref), converged=st["converged"])


def test_twin_entry_points_are_the_same_solve(B, O):
    """The reference's _v2 / _nooverlap twins (bit-identical there, tests/test_oracle_golden_shifted_lop.py) map to the same solve."""
    B.set_options(quiet=1, cache=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    case = SHIFTED_LOP_CASES[0]
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    out = {}
    for v in SHIFTED_LOP_VARIANTS:
        x = np.zeros((sigma.size, n)); r = b.copy()
        ret = getattr(B.lib, v)(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), x.ctypes.data, r.ctypes.data,
                                np.ascontiguousarray(sigma).ctypes.data, sigma.size, seed)
        out[v] = (ret, x, r)
    for a, b_ in (("shifted_lopbicgstab", "shifted_lopbicgstab_v2"), ("shifted_lopbicgstab", "shifted_lopbicgstab_nooverlap"),
                  ("shifted_pipe_lopbicgstab", "shifted_pipe_lopbicgstab_nooverlap")):
        assert out[a][0] == out[b_][0]
        assert np.abs(out[a][1] - out[b_][1]).max() <= 1e-12 * np.abs(out[a][1]).max()


@pytest.mark.parametrize("algo,pipe", ALGOS)
def test_shifted_lop_stdout_contract(B, O, capfd, algo, pipe):
    case = SHIFTED_LOP_CASES[0]
    B.set_options(quiet=0, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    x = np.zeros((sigma.size, n)); r = b.copy()
    ret = _entry(B, pipe)(blk, x, r, sigma, seed)
    B.lib.bicg_synchronize()
    C.CDLL(None).fflush(None)
    out = capfd.readouterr().out
    B.set_options(quiet=1)
    assert f"Total iter   : {ret}\n" in out                                           # shifted_solver.c:340 / :883
    fr = float(re.search(r"Final r      : (\S+)", out).group(1))                     # :341 / :884
    assert abs(fr - np.sqrt(B.last_history()[ret])) <= 1e-6 * fr
    assert "Total time   : " in out and " [sec.] \n" in out and "Avg time/iter: " in out


@pytest.mark.parametrize("algo,pipe", ALGOS)
@pytest.mark.parametrize("L,seed", [(1, 0), (5, 2), (5, 4)])
def test_shifted_lop_seed_only_and_other_seeds(B, O, algo, pipe, L, seed):
    B.set_options(quiet=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, "stencil15", 12, 14.0)
    sigma = np.arange(L) * 0.01 + 0.01
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[seed], np.ones(n), b)
    ref = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, tol=1e-12, max_iter=MAX_ITER)
    x = np.zeros((L, n)); r = b.copy()
    ret = _entry(B, pipe)(blk, x, r, sigma, seed)
    _check(O, n, ptr, col, val, sigma, b, ret, x, r, B.last_history(), ref, what=(algo, L, seed))
    assert np.abs(x[seed] - 1.0).max() < 1e-8


def test_shifted_solve_ex_and_argument_checks(B, O):
    """bicg_shifted_solve_ex on a resident matrix: each method is the solve of its reference entry point; bad arguments give -1."""
    B.set_options(quiet=1, cache=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    case = SHIFTED_LOP_CASES[0]
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    dm = B.DeviceMatrix(blk)
    for method, pipe in (("shifted_lopbicgstab", False), ("shifted_pipe_lopbicgstab", True)):
        ref = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, tol=1e-12, max_iter=MAX_ITER)
        x = np.zeros((sigma.size, n)); r = b.copy()
        ret, st = dm.shifted_solve(method, x, r, sigma, seed)
        assert st["iters"] == ret and st["kernel_launches"] > 0 and st["loop_ms"] > 0
        _check(O, n, ptr, col, val, sigma, b, ret, x, r, B.last_history(), ref, what=method)
    x = np.zeros((sigma.size, n)); r = b.copy()
    ret, st = dm.shifted_solve("shifted_lopbicg_switching", x, r, sigma, seed)
    assert ret == st["iters"] + 1 and abs(ret - O.shifted_solve(n, ptr, col, val, b, sigma, seed)["ret"]) <= 2
    x = np.zeros((sigma.size, n)); r = b.copy(); sg = np.ascontiguousarray(sigma)
    for method, L, sd in ((1, 0, 0), (2, sigma.size, sigma.size), (1, sigma.size, -1), (7, sigma.size, 0)):
        assert B.lib.bicg_shifted_solve_ex(dm.h, method, x.ctypes.data, r.ctypes.data, sg.ctypes.data, L, sd, None) == -1
    for v in SHIFTED_LOP_VARIANTS:
        assert getattr(B.lib, v)(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), x.ctypes.data, r.ctypes.data, sg.ctypes.data,
                                 0, 0) == -1
    dm.destroy()


@pytest.mark.parametrize("algo,pipe", ALGOS)
def test_shifted_lop_many_shifts_medium_size(B, O, algo, pipe):
    """64 shifts on a 250 k-row matrix (T' family, 63^3): the fused multi-shift pass with a full coefficient table.  The
    iteration count to 1e-10 is chaotic in the summation order of the dots: the oracle's own P = 1, 2, 3, 4, 8 emulations stop
    after 157 - 176 iterations (LOP) and 152 - 282 (PIPE-LOP).  LOP stops when the seed's own BiCGStab residual reaches the
    tolerance (every other shift's |1/(zeta pi)| is below 1 here), so its count is as chaotic as plain BiCGStab's on this
    matrix; an H100 SXM (132 SMs) took 181 and 186 in two runs, whose SpMV configurations the autotuner picked by timing.  The
    count is held to max(2, 10 %) around the spread of the oracle's P = 1, 2, 4, 8 runs; the history of the first 10
    iterations and every sampled x_j against its own shifted system are held as in the other tests."""
    B.set_options(quiet=1, shift_tol=1e-10, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, "stencil15", 63, 14.0)
    L, seed = 64, 0
    sigma = (np.arange(L) + 1) * (0.5 / L)
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[seed], np.ones(n), b)
    refs = [OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, P=P, tol=1e-10, max_iter=MAX_ITER) for P in (1, 2, 4, 8)]
    x = np.zeros((L, n)); r = b.copy()
    ret = _entry(B, pipe)(blk, x, r, sigma, seed)
    hist = B.last_history()
    B.set_options(shift_tol=1e-12)
    rets = [f["ret"] for f in refs]
    assert max(rets) < MAX_ITER, rets                                               # the case does converge
    lo, hi = min(rets), max(rets)
    assert lo - max(2, int(0.1 * lo)) <= ret <= hi + max(2, int(0.1 * hi)), (ret, rets)
    m = min(10, ret, lo)
    got, want = np.sqrt(hist[1:m + 1]), np.sqrt(refs[0]["hist"][1:m + 1])
    assert np.all(np.abs(got - want) <= 1e-10 * want + 1e-15)
    for j in (0, 1, 31, 63):
        res = np.linalg.norm(O.spmv(n, ptr, col, val, x[j]) + sigma[j] * x[j] - b)
        res_ref = np.linalg.norm(O.spmv(n, ptr, col, val, refs[0]["x"][j]) + sigma[j] * refs[0]["x"][j] - b)
        assert res <= max(10 * res_ref, 1e-8 * np.linalg.norm(b)), (j, res, res_ref)


@pytest.mark.parametrize("algo,pipe", ALGOS)
def test_shifted_lop_512_shifts(B, O, algo, pipe):
    """main_shifted.c's 512 shifts on a small matrix: the whole coefficient table of the fused pass in shared memory."""
    B.set_options(quiet=1, shift_tol=1e-12, shift_max_iter=MAX_ITER)
    blk, n, ptr, col, val = global_csr(B, "stencil15", 12, 14.0)
    L, seed = 512, 0
    sigma = (np.arange(L) + 1) * (0.01 / L)
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[seed], np.ones(n), b)
    ref = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=pipe, tol=1e-12, max_iter=MAX_ITER)
    x = np.zeros((L, n)); r = b.copy()
    ret = _entry(B, pipe)(blk, x, r, sigma, seed)
    _check(O, n, ptr, col, val, sigma, b, ret, x, r, B.last_history(), ref, what=(algo, L))


def test_unchanged_test_shifted_driver(tmp_path):
    """The reference's test_shifted.c, UNCHANGED, linked against the library (oracle/_ref/ref_test_shifted_b200, built where a
    checkout of the reference exists): its `Total iter` on the golden .mtx file within 2 of what the reference's own build printed."""
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_test_shifted_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_test_shifted_b200 not built")
    gold = int(np.load(golden_path("shifted_pipe_lopbicgstab_nooverlap"))["test_shifted_mtx|total_iter"])
    p = subprocess.run([exe, mtx_path()], capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "Node: 1, Proc: 1" in p.stdout
    it = int(re.search(r"Total iter\s*:\s*(\d+)", p.stdout).group(1))
    assert abs(it - gold) <= 2, (it, gold)
