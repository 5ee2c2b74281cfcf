"""CPU: the oracle's restatement of shifted_lopbicg (shifted_switching_solver.c:20-257, oracle/shifted_fixed_oracle.c) is
bit-identical to what the reference's own compiled function produced (tests/golden/ref_shifted_fixed.npz, generator
tests/golden/make_golden_shifted_fixed.py): return value, every x_j, the seed residual r and the residual history.  And until the
seed converges, the fixed-seed solver is the switching one: the restatements of both give the same bits up to the first switch."""
import hashlib

import numpy as np
import pytest
import shifted_fixed_oracle as OF

from helpers import X0_GOLDEN, X0_SHIFTED_MAX_ITER, X0_SHIFTED_TOL, global_csr, x0_shifted_problem
from shifted_fixed_cases import FIXED_CASES, FIXED_LARGE_CASES, GOLDEN_FIXED, fixed_problem


def _gold(name):
    g = np.load(GOLDEN_FIXED)
    return {k.split("|")[1]: g[k] for k in g.files if k.split("|")[0] == name}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


@pytest.mark.parametrize("case", FIXED_CASES + FIXED_LARGE_CASES, ids=[c[0] for c in FIXED_CASES + FIXED_LARGE_CASES])
def test_oracle_matches_reference_bitwise(B, O, case):
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    got = OF.shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=1000)
    want = _gold(case[0])
    assert got["ret"] == int(want["ret"])
    assert np.array_equal(np.sqrt(got["hist"][1:]), want["res"])        # the reference prints every iteration (OUT_ITER = 1)
    if "x" in want:
        assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["r"], want["r"])
    else:
        assert _sha(got["x"]) == str(want["x_sha256"]) and _sha(got["r"]) == str(want["r_sha256"])
    # every shift stopped, at most at the last iteration, and a stop iteration is 1-based
    assert np.all(got["stop_iter"] >= 1) and got["stop_iter"].max() == got["ret"]


@pytest.mark.parametrize("case", FIXED_CASES, ids=[c[0] for c in FIXED_CASES])
def test_fixed_and_switching_share_the_prefix(B, O, case):
    """Up to the first seed switch (the iteration at which the seed stopped while other shifts had not), the restatements of
    shifted_lopbicg and shifted_lopbicg_switching give the same history and stop the same shifts at the same iterations with
    the same x_j.  Without a switch they are the same solve and the fixed one returns one less."""
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    fx = OF.shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=1000)
    sw = O.shifted_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=1000)
    k_s = int(fx["stop_iter"][seed])
    assert k_s == sw["stop_iter"][seed]
    if k_s == fx["ret"]:                                                  # the seed stopped last: no switch
        assert sw["seed"] == seed and sw["ret"] == fx["ret"] + 1
        assert np.array_equal(fx["hist"], sw["hist"]) and np.array_equal(fx["x"], sw["x"]) and np.array_equal(fx["r"], sw["r"])
        assert np.array_equal(fx["stop_iter"], sw["stop_iter"])
        return
    assert sw["seed"] != seed and fx["ret"] > k_s                        # the fixed seed kept iterating past its own stop
    assert np.array_equal(fx["hist"][:k_s + 1], sw["hist"][:k_s + 1])
    assert not np.array_equal(fx["hist"][k_s + 1:k_s + 2], sw["hist"][k_s + 1:k_s + 2])
    early = [j for j in range(sigma.size) if j != seed and 0 < fx["stop_iter"][j] <= k_s]
    for j in early:
        assert fx["stop_iter"][j] == sw["stop_iter"][j] and np.array_equal(fx["x"][j], sw["x"][j]), j
    late = [j for j in range(sigma.size) if fx["stop_iter"][j] > k_s]
    assert all(sw["stop_iter"][j] > k_s for j in late)


@pytest.mark.parametrize("case", FIXED_CASES, ids=[c[0] for c in FIXED_CASES])
def test_fixed_solves_every_shifted_system(B, O, case):
    """Every x_j the reference's shifted_lopbicg returns solves (A + sigma_j I) x_j = b to EPS, including on the cases whose seed
    converges first and keeps iterating."""
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    x = _gold(case[0])["x"]
    for j in range(sigma.size):
        res = O.spmv(n, ptr, col, val, x[j]) + sigma[j] * x[j] - b
        assert np.linalg.norm(res) <= 10 * tol * np.linalg.norm(b), (j, np.linalg.norm(res) / np.linalg.norm(b))


def test_oracle_from_nonzero_x0_matches_reference_bitwise(B, O):
    """From a nonzero x_set (tests/golden/ref_x0.npz): the reference's return value, every x_j, r and printed residual."""
    gold = np.load(X0_GOLDEN)
    n, ptr, col, val, b, sigma, seed, x0 = x0_shifted_problem(B, O, gold)
    got = OF.shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, tol=X0_SHIFTED_TOL, max_iter=X0_SHIFTED_MAX_ITER, x0=x0)
    want = {k: gold[f"shifted|shifted_lopbicg|{k}"] for k in ("ret", "res", "x", "r")}
    assert got["ret"] == want["ret"]
    assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["r"], want["r"])
    assert np.array_equal(np.sqrt(got["hist"][1:]), want["res"])
