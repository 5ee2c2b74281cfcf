"""tests/shifted_loop_reference.py against the C oracles (no GPU): run to the end of a solve, the restated shifted solvers must
give the oracles' return value, every x_j, the seed residual r, the residual history, the final seed and every stop iteration
bit for bit, for all four methods.  The oracles are pinned to the compiled reference (test_oracle_golden*.py), so this pins the
restatement that tests/test_gpu_shifted_state.py compares the GPU with after every iteration."""
import numpy as np
import pytest
import shifted_fixed_oracle as OF
import shifted_lop_oracle as OL

from helpers import global_csr, initial_x_set
from shifted_fixed_cases import FIXED_CASES, FIXED_LARGE_CASES, fixed_problem
from shifted_loop_reference import METHODS, shifted_reference_solve, shifted_reference_states

MAX_ITER = 1000
CASES = FIXED_CASES + FIXED_LARGE_CASES[:1]          # every SHIFTED_LOP_CASES entry, L = 1, seeds 0 / middle / last; 512 shifts


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def oracle_solve(O, method, n, ptr, col, val, b, sigma, seed, tol, max_iter, x0=None):
    """The C oracle of `method` at P = 1 from the initial x_set x0 (None: zero): dict(ret, x, r, hist, seed, stop_iter); seed /
    stop_iter are None where the oracle does not report them (the LOP family neither switches nor stops single shifts)."""
    if method == "shifted_lopbicg_switching":
        out = O.shifted_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=max_iter, x0=x0)
        return dict(ret=out["ret"], x=out["x"], r=out["r"], hist=out["hist"], seed=out["seed"], stop_iter=out["stop_iter"])
    if method == "shifted_lopbicg":
        out = OF.shifted_fixed_solve(n, ptr, col, val, b, sigma, seed, tol=tol, max_iter=max_iter, x0=x0)
        return dict(ret=out["ret"], x=out["x"], r=out["r"], hist=out["hist"], seed=seed, stop_iter=out["stop_iter"])
    out = OL.shifted_lop_solve(n, ptr, col, val, b, sigma, seed, pipe=method == "shifted_pipe_lopbicgstab", tol=tol, max_iter=max_iter,
                               x0=x0)
    return dict(ret=out["ret"], x=out["x"], r=out["r"], hist=out["hist"], seed=None, stop_iter=None)


def assert_same_as_oracle(got, ret, want, what):
    assert ret == want["ret"], (what, ret, want["ret"])
    assert _bits(got["hist"]) == _bits(want["hist"]), (what, "hist")
    assert _bits(got["r"]) == _bits(want["r"]), (what, "r")
    for j in range(want["x"].shape[0]):
        assert _bits(got["x"][j]) == _bits(want["x"][j]), (what, "x", j)
    if want["seed"] is not None:
        assert got["seed"] == want["seed"], (what, got["seed"], want["seed"])
        assert np.array_equal(got["stop_iter"], want["stop_iter"]), (what, got["stop_iter"], want["stop_iter"])


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_restatement_bitwise_equal_to_oracle(B, O, case, method):
    _, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    want = oracle_solve(O, method, n, ptr, col, val, b, sigma, seed, tol, MAX_ITER)
    got, ret = shifted_reference_solve(O, method, ptr, col, val, b, sigma, seed, tol, MAX_ITER)
    assert_same_as_oracle(got, ret, want, (case[0], method))
    if method == "shifted_lopbicg_switching" and case[0].endswith("_switch"):
        assert any(d[0] == "switch" for d in got["decisions"]), got["decisions"]      # the seed does switch here


X0_CASES = [c for c in FIXED_CASES if c[0] in ("sh_stencil15_g12_L5", "sh_convdiff_g40_L6_switch", "fx_stencil15_g12_L5_seed2")]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", X0_CASES, ids=[c[0] for c in X0_CASES])
def test_restatement_from_nonzero_x0_bitwise_equal_to_oracle(B, O, case, method):
    """The shifted solvers never form b - A x0: they only add to each x_j, so a nonzero initial x_set carries through to the
    result, and the restatement must still give the oracles' bits, through the seed switch of the _switch case too."""
    _, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, tol = fixed_problem(O, n, ptr, col, val, case)
    x0 = initial_x_set(sigma.size, n)
    want = oracle_solve(O, method, n, ptr, col, val, b, sigma, seed, tol, MAX_ITER, x0=x0)
    got, ret = shifted_reference_solve(O, method, ptr, col, val, b, sigma, seed, tol, MAX_ITER, x0=x0)
    assert_same_as_oracle(got, ret, want, (case[0], method, "x0"))
    zero = oracle_solve(O, method, n, ptr, col, val, b, sigma, seed, tol, MAX_ITER)
    assert want["ret"] == zero["ret"] and _bits(want["hist"]) == _bits(zero["hist"])     # x0 changes nothing but x
    assert not np.array_equal(want["x"], zero["x"])
    if method == "shifted_lopbicg_switching" and case[0].endswith("_switch"):
        assert any(d[0] == "switch" for d in got["decisions"]), got["decisions"]


def _switch_iteration(O, B, case, tol):
    _, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, _ = fixed_problem(O, n, ptr, col, val, case)
    st = shifted_reference_states(O, "shifted_lopbicg_switching", ptr, col, val, b, sigma, seed, [200], tol=tol, keep_p=False)[200]
    return [d[1] for d in st["decisions"] if d[0] == "switch"]


@pytest.mark.parametrize("tol", [1e-12, 1e-6])
@pytest.mark.parametrize("method", METHODS)
def test_states_are_prefixes_of_one_run(B, O, method, tol):
    """shifted_reference_states() keeps the states of one pass; each equals the oracle run with max_iter = k, which pins each
    solver's max_iter semantics (the switching solver returns iterations + 1, the others the iterations performed).  The
    case switches its seed; the iterations around the switch are among the k."""
    case = next(c for c in FIXED_CASES if c[0] == "sh_convdiff_g40_L6_switch")
    _, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed, _ = fixed_problem(O, n, ptr, col, val, case)
    ks_switch = _switch_iteration(O, B, case, tol)
    assert ks_switch, "the case must switch its seed"
    ks = sorted({1, 2, 3, 7, 8, 9, 17} | {k for s in ks_switch[:1] for k in (s - 1, s, s + 1, s + 2)})
    states = shifted_reference_states(O, method, ptr, col, val, b, sigma, seed, ks, tol=tol)
    assert sorted(states) == ks
    for k, st in states.items():
        want = oracle_solve(O, method, n, ptr, col, val, b, sigma, seed, tol, k)
        assert_same_as_oracle(st, st["ret"], want, (method, k))
        assert st["iters"] <= k and st["hist"].size == st["iters"] + 1
        assert st["ret"] == st["iters"] + (1 if method == "shifted_lopbicg_switching" else 0)
