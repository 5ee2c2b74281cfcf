"""CPU: the oracle restatement (oracle/bicg_oracle.c) against the golden vectors the REFERENCE produced
(tests/golden/ref_histories_P*.npz, generator tests/golden/make_golden.py) -- bit for bit, for 1, 2 and 3 ranks --
and against further outputs of the compiled reference (tests/golden/ref_live.npz, tests/golden/make_golden_live.py; from
nonzero initial guesses tests/golden/ref_x0.npz, tests/golden/make_golden_x0.py)."""
import os

import numpy as np
import pytest

from helpers import (METHODS, RR, SMALL_CASES, X0_GOLDEN, X0_KINDS, X0_PLAIN, X0_PLAIN_MAX_ITER, X0_PLAIN_TOL, X0_RR, global_csr,
                     initial_guess)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL, MAX_ITER = 1e-10, 600


@pytest.fixture(scope="module")
def gold():
    out = {}
    for P in (1, 2, 3):
        out.update(np.load(os.path.join(GOLDEN, f"ref_histories_P{P}.npz")))
    return out


@pytest.fixture(scope="module")
def gold_live():
    return np.load(os.path.join(GOLDEN, "ref_live.npz"))


@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("name,kind,g,p0", SMALL_CASES)
def test_oracle_reproduces_reference_bitwise(B, O, gold, name, kind, g, p0, P):
    blk, n, ptr, col, val = global_csr(B, kind, g, p0)
    b = O.spmv(n, ptr, col, val, np.ones(n), P=P)              # main.c:109-113 with P ranks
    for method in METHODS:
        kw = RR if method.endswith("rr") else {}
        o = O.solve(method, n, ptr, col, val, b, P=P, tol=TOL, max_iter=MAX_ITER, **kw)
        key = f"{name}|{method}|P{P}"
        assert o["iters"] == int(gold[key + "|iters"]), key
        assert np.array_equal(np.sqrt(o["hist"][1:]), gold[key + "|res"]), key      # every iteration, every bit
        assert np.array_equal(o["x"], gold[key + "|x"]), key
        assert np.array_equal(o["r"], gold[key + "|r"]), key


def test_oracle_against_compiled_reference_live(B, O, gold_live):
    blk, n, ptr, col, val = global_csr(B, "convdiff", 25, 2.0, seed=99)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    for method in METHODS:
        kw = dict(krr=7, nrr=2) if method.endswith("rr") else {}
        o = O.solve(method, n, ptr, col, val, b, tol=1e-11, max_iter=400, **kw)
        r = {k: gold_live[f"cd25|{method}|{k}"] for k in ("iters", "res", "x", "r")}
        assert o["iters"] == r["iters"]
        assert np.array_equal(np.sqrt(o["hist"][1:]), r["res"])
        assert np.array_equal(o["x"], r["x"]) and np.array_equal(o["r"], r["r"])


@pytest.fixture(scope="module")
def gold_x0():
    return np.load(X0_GOLDEN)


@pytest.mark.parametrize("x0_kind", X0_KINDS)
def test_oracle_from_nonzero_x0_against_compiled_reference(B, O, gold_x0, x0_kind):
    """From x0 != 0 (solver.c:74-83: r0 = b - A x0, r# = r0, dot_zero = (r0, r0); pipe_bicgstab_rr keeps the caller's b for its
    replacements, :475 / :524) the oracle gives the reference's iteration count, every printed residual, x and r bit for bit."""
    kind, g, p0, gseed = X0_PLAIN
    _, n, ptr, col, val = global_csr(B, kind, g, p0, seed=gseed)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    x0 = gold_x0[f"plain|{x0_kind}|x0"]
    assert np.array_equal(x0, initial_guess(x0_kind, n))
    for method in METHODS:
        kw = X0_RR if method == "pipe_bicgstab_rr" else {}
        o = O.solve(method, n, ptr, col, val, b, x0=x0, tol=X0_PLAIN_TOL, max_iter=X0_PLAIN_MAX_ITER, **kw)
        r = {k: gold_x0[f"plain|{x0_kind}|{method}|{k}"] for k in ("iters", "res", "x", "r")}
        assert 0 < o["iters"] == r["iters"] < X0_PLAIN_MAX_ITER, (method, o["iters"], r["iters"])
        assert np.array_equal(np.sqrt(o["hist"][1:]), r["res"]), method
        assert np.array_equal(o["x"], r["x"]) and np.array_equal(o["r"], r["r"]), method


def test_oracle_rhs_ones_multi_rank_live(B, O, gold_live):
    """README / BASELINE wording "right-hand side = all ones" (main.c itself uses b = A*1): the oracle follows the
    compiled reference for that rhs too, with 1 and 3 ranks."""
    blk, n, ptr, col, val = global_csr(B, "stencil15", 9, 14.0)
    for P in (1, 3):
        for method in METHODS[:3]:
            o = O.solve(method, n, ptr, col, val, np.ones(n), P=P, tol=1e-11, max_iter=400)
            r = {k: gold_live[f"ones|{method}|P{P}|{k}"] for k in ("iters", "res", "x", "r")}
            assert o["iters"] == r["iters"]
            assert np.array_equal(np.sqrt(o["hist"][1:]), r["res"])
            assert np.array_equal(o["x"], r["x"]) and np.array_equal(o["r"], r["r"])


def test_oracle_spmv_and_blas1(B, O):
    blk, n, ptr, col, val = global_csr(B, "random", 500, 6)
    import scipy.sparse as sp
    A = sp.csr_matrix((val, col, ptr), shape=(n, n))
    x = np.random.default_rng(1).standard_normal(n)
    for P in (1, 2, 5):
        assert np.allclose(O.spmv(n, ptr, col, val, x, P=P), A @ x, rtol=1e-13, atol=1e-13)
    assert np.allclose(O.spmv(n, ptr, col, val, x, long_double=True), A @ x, rtol=1e-13, atol=1e-13)
    y = np.random.default_rng(2).standard_normal(n)
    assert abs(O.lib().orc_ddot(n, x.ctypes.data_as(O._dp), y.ctypes.data_as(O._dp)) - float(x @ y)) < 1e-12


def test_manufactured_solution(B, O):
    """x* = 1 (main.c:109-117): every variant recovers it."""
    blk, n, ptr, col, val = global_csr(B, "stencil15", 9, 14.0)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    for method in METHODS:
        kw = RR if method.endswith("rr") else {}
        o = O.solve(method, n, ptr, col, val, b, tol=1e-12, max_iter=500, **kw)
        assert np.abs(o["x"] - 1).max() < 1e-8


# ---- shifted family (SURVEY.md 8(f) N4) --------------------------------------------------------------------------
from helpers import SHIFTED_CASES, X0_SHIFTED_MAX_ITER, X0_SHIFTED_TOL, shifted_problem, x0_shifted_problem


@pytest.fixture(scope="module")
def gold_shifted():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shifted.npz"))


@pytest.mark.parametrize("name,kind,g,p0,L,scale,seed", SHIFTED_CASES)
def test_shifted_oracle_reproduces_reference_bitwise(B, O, gold_shifted, name, kind, g, p0, L, scale, seed):
    """orc_shifted_lopbicg_switching vs the golden outputs of the reference's own shifted_lopbicg_switching
    (shifted_switching_solver.c:260-602, strict build): same return value, bit-identical x_j for every shift, r and history."""
    blk, n, ptr, col, val = global_csr(B, kind, g, p0)
    sigma, b = shifted_problem(O, n, ptr, col, val, L, scale, seed)
    o = O.shifted_solve(n, ptr, col, val, b, sigma, seed, tol=1e-12, max_iter=1000)
    assert o["ret"] == int(gold_shifted[name + "|ret"])
    assert np.array_equal(o["x"], gold_shifted[name + "|x"])
    assert np.array_equal(o["r"], gold_shifted[name + "|r"])
    assert np.array_equal(np.sqrt(o["hist"][1:]), gold_shifted[name + "|res"])
    if "switch" in name:
        assert o["seed"] != seed                                   # the seed-switching branch really ran
    for j in range(L):                                             # and every shifted system is solved
        res = O.spmv(n, ptr, col, val, o["x"][j]) + sigma[j] * o["x"][j] - b
        assert np.linalg.norm(res) <= 1e-10 * np.linalg.norm(b)


@pytest.mark.parametrize("name,kind,g,p0,L,scale,seed", SHIFTED_CASES)
def test_reference_noovlp_twin_is_the_same_solve(B, O, gold_shifted, gold_live, name, kind, g, p0, L, scale, seed):
    """shifted_lopbicg_switching_noovlp (shifted_switching_solver.c:611) differs from shifted_lopbicg_switching only in when it waits
    for the halo exchange and in its timers: return value, every x_j, r and the residual history of the two compiled reference
    functions (golden outputs of each) are bit-identical -- which is why the library exports the former as the latter
    (csrc/abi.cu) -- and the oracle reproduces the twin too."""
    a = {k: gold_shifted[f"{name}|{k}"] for k in ("ret", "x", "r", "res")}
    c = {k: gold_live[f"noovlp|{name}|{k}"] for k in ("ret", "x", "r", "res")}
    blk, n, ptr, col, val = global_csr(B, kind, g, p0)
    sigma, b = shifted_problem(O, n, ptr, col, val, L, scale, seed)
    o = O.shifted_solve(n, ptr, col, val, b, sigma, seed)
    assert o["ret"] == c["ret"] and np.array_equal(o["x"], c["x"]) and np.array_equal(o["r"], c["r"])
    assert np.array_equal(np.sqrt(o["hist"][1:]), c["res"])
    assert a["ret"] == c["ret"] and np.array_equal(a["x"], c["x"]) and np.array_equal(a["r"], c["r"])
    assert np.array_equal(a["res"], c["res"])


def test_shifted_oracle_from_nonzero_x0_against_compiled_reference(B, O, gold_x0):
    """orc_shifted_lopbicg_switching from a nonzero x_set, through a seed switch: the reference's return value, every x_j, r and
    printed residual, bit for bit.  The solver only adds to each x_j, so x0 reaches the result."""
    n, ptr, col, val, b, sigma, seed, x0 = x0_shifted_problem(B, O, gold_x0)
    o = O.shifted_solve(n, ptr, col, val, b, sigma, seed, tol=X0_SHIFTED_TOL, max_iter=X0_SHIFTED_MAX_ITER, x0=x0)
    want = {k: gold_x0[f"shifted|shifted_lopbicg_switching|{k}"] for k in ("ret", "res", "x", "r")}
    assert o["ret"] == want["ret"] and o["seed"] != seed
    assert np.array_equal(o["x"], want["x"]) and np.array_equal(o["r"], want["r"])
    assert np.array_equal(np.sqrt(o["hist"][1:]), want["res"])
