"""tests/loop_reference.py against the oracle (no GPU): run to the end of a solve, the restated loops must give the oracle's
iteration count, x, r and residual history bit for bit, for all four methods and replacement periods from every iteration
to every tenth, from x0 = 0 and from nonzero initial guesses.  The oracle is pinned to the compiled reference
(test_oracle_golden.py), so this pins the restatement that the per-iteration GPU tests compare with."""
import numpy as np
import pytest

from helpers import METHODS, SMALL_CASES, X0_KINDS, global_csr, initial_guess
from loop_reference import reference_state, reference_states

TOL, MAX_ITER = 1e-10, 1000


def _variants():
    for method in METHODS:
        if method == "pipe_bicgstab_rr":
            for krr in (1, 2, 3, 10):
                yield pytest.param(method, krr, 3, id=f"{method}-krr{krr}")
        else:
            yield pytest.param(method, 0, 0, id=method)


@pytest.mark.parametrize("method,krr,nrr", list(_variants()))
@pytest.mark.parametrize("name,kind,g,p0", SMALL_CASES, ids=[c[0] for c in SMALL_CASES])
def test_restatement_bitwise_equal_to_oracle(B, O, name, kind, g, p0, method, krr, nrr):
    _, n, ptr, col, val = global_csr(B, kind, g, p0)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    want = O.solve(method, n, ptr, col, val, b, tol=TOL, max_iter=MAX_ITER, krr=krr, nrr=nrr)
    got = reference_state(O, method, ptr, col, val, b, MAX_ITER, krr=krr, nrr=nrr, tol=TOL)
    assert 0 < want["iters"] < MAX_ITER                        # the solve converged: the tolerance test ended both
    assert got["iters"] == want["iters"]
    assert np.array_equal(got["hist"], want["hist"])
    assert np.array_equal(got["x"], want["x"])
    assert np.array_equal(got["r"], want["r"])


@pytest.mark.parametrize("method", METHODS)
def test_states_are_prefixes_of_one_run(B, O, method):
    """reference_states() keeps the states of one pass; each equals a run stopped at that k by max_iter."""
    _, n, ptr, col, val = global_csr(B, "convdiff", 40, 1.5)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    kw = dict(krr=2, nrr=2) if method.endswith("rr") else {}
    states = reference_states(O, method, ptr, col, val, b, [1, 3, 6], **kw)
    assert sorted(states) == [1, 3, 6]
    for k, st in states.items():
        one = reference_state(O, method, ptr, col, val, b, k, **kw)
        ref = O.solve(method, n, ptr, col, val, b, tol=0.0, max_iter=k, **kw)
        assert st["iters"] == one["iters"] == ref["iters"] == k
        assert np.array_equal(st["hist"], ref["hist"])
        for name in st:
            assert np.array_equal(st[name], one[name]), name
        assert np.array_equal(st["x"], ref["x"]) and np.array_equal(st["r"], ref["r"])


@pytest.mark.parametrize("x0_kind", X0_KINDS)
@pytest.mark.parametrize("method,krr,nrr", list(_variants()))
@pytest.mark.parametrize("name,kind,g,p0", SMALL_CASES, ids=[c[0] for c in SMALL_CASES])
def test_restatement_from_nonzero_x0_bitwise_equal_to_oracle(B, O, name, kind, g, p0, method, krr, nrr, x0_kind):
    """From x0 != 0 the init computes r0 = b - A x0, r# = r0 and dot_zero = (r0, r0), and pipe_bicgstab_rr keeps the caller's b
    for its replacements: none of these equals b, as they all do from x0 = 0."""
    _, n, ptr, col, val = global_csr(B, kind, g, p0)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    x0 = initial_guess(x0_kind, n)
    want = O.solve(method, n, ptr, col, val, b, x0=x0, tol=TOL, max_iter=MAX_ITER, krr=krr, nrr=nrr)
    got = reference_state(O, method, ptr, col, val, b, MAX_ITER, krr=krr, nrr=nrr, tol=TOL, x0=x0)
    assert 0 < want["iters"] < MAX_ITER
    assert got["iters"] == want["iters"]
    assert np.array_equal(got["hist"], want["hist"])
    assert np.array_equal(got["x"], want["x"])
    assert np.array_equal(got["r"], want["r"])
    if method == "pipe_bicgstab_rr" and krr > 0:
        assert np.array_equal(got["b"], b)                            # the caller's b, not r0
