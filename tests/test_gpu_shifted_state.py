"""Every shifted solver held to the reference iteration by iteration (-m gpu): shifted_lopbicg_switching, shifted_lopbicg,
shifted_lopbicgstab and shifted_pipe_lopbicgstab.

A solve with shift_max_iter = k stops after iteration k (or where its own tolerance test stops it first); then its return
value, iteration count, history, final seed, every shift's stop iteration, every x_j of every shift and the seed residual r
are compared with tests/shifted_loop_reference.py stopped at the same k.  The counts must match exactly.  Vectors and history
are held by the rule of tests/state_check.py: at most max(FLOOR, FACTOR * spread), the spread being the distance between the
restatement and its exact evaluation; each x_j and r to its own spread, the history to the largest spread among its entries.
A case whose two evaluations take different stop or switch decisions up to the last k says nothing about the kernels and is
refused, as is one whose spread exceeds MAX_SPREAD.

The k straddle the host's batches of U = 8 iterations with DEPTH = 2 of them enqueued ahead of the done flag (a batch that
runs past the done flag must not move anything), the seed switch (k_s - 1 .. k_s + 2, k_s taken from the restatement), and a
shift that has stopped must not move at all: its x_j stays bit-identical from its stop iteration on.

Shapes: every method on the shifted cases (seeds 0, middle and last), n = 17, 2111 and a ragged matrix, L = 1, 2, 33,
512, 513, both sides of the shift counts at which the update kernels' coefficient tables outgrow the 48 KB of shared memory a
block gets by default (they then take the shifts in passes), 8192 shifts, every forced stand-alone SpMV variant (its shifted
epilogue under the 0-, 1- and 2-dot epilogues) and a 216 k-row matrix with 64 shifts."""
import numpy as np
import pytest

from helpers import global_csr, initial_x_set, shifted_problem
from shifted_fixed_cases import FIXED_CASES
from shifted_loop_reference import METHODS, shifted_reference_states
from state_check import MATRICES, STANDALONE, _hold, _rel, matrix

pytestmark = pytest.mark.gpu

KS = (1, 2, 3, 7, 8, 9, 17)
SWITCHING, FIXED = "shifted_lopbicg_switching", "shifted_lopbicg"
LOP = ("shifted_lopbicgstab", "shifted_pipe_lopbicgstab")
DEFAULTS = dict(quiet=1, shift_tol=1e-12, shift_max_iter=1000, shift_error=0, spmv="auto", spmv_lanes=0, spmv_threads=0,
                spmv_stages=0, autotune=1)


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(**(DEFAULTS | dict(autotune=0)))
    yield
    B.set_options(**DEFAULTS)


# ---- problems -------------------------------------------------------------------------------------------------------
def _matrix(B, spec):
    """A state_check.MATRICES name, or (kind, g, p0) of the generator."""
    if isinstance(spec, str):
        return matrix(B, spec)
    _, n, ptr, col, val = global_csr(B, *spec)
    return n, ptr, col, val


def _problem(O, n, ptr, col, val, L, scale, seed):
    """sigma_j = (j + 1) scale (scale None: test_shifted.c's 0.01 j + 0.01) and b = (A + sigma_seed I) 1."""
    if scale is not None:
        return shifted_problem(O, n, ptr, col, val, L, scale, seed)
    sigma = np.arange(L) * 0.01 + 0.01
    b = O.spmv(n, ptr, col, val, np.ones(n))
    O.daxpy(sigma[seed], np.ones(n), b)
    return sigma, b


_REF = {}


def reference(B, O, spec, method, L, scale, seed, tol, ks, keep_p=True, x0=False):
    """(restatement states, exact-evaluation states) for ks, once per matrix, method, tolerance, shift set, seed and initial
    x_set (x0: helpers.initial_x_set instead of zero)."""
    key = (str(spec), method, L, scale, seed, tol, tuple(ks), x0)
    if key not in _REF:
        n, ptr, col, val = _matrix(B, spec)
        sigma, b = _problem(O, n, ptr, col, val, L, scale, seed)
        xs = initial_x_set(L, n) if x0 else None
        _REF[key] = tuple(shifted_reference_states(O, method, ptr, col, val, b, sigma, seed, ks, tol=tol, exact=e, keep_p=keep_p, x0=xs)
                          for e in (False, True))
        if n * L > 1 << 22:                        # the 216 k-row case: its states are not kept
            return _REF.pop(key)
    return _REF[key]


def switch_iteration(B, O, spec, L, scale, seed, tol):
    """The first seed switch of the switching solver, from the restatement (None: no switch in 40 iterations)."""
    st = reference(B, O, spec, SWITCHING, L, scale, seed, tol, (40,), keep_p=False)[0][40]
    return next((d[1] for d in st["decisions"] if d[0] == "switch"), None)


# ---- comparison -----------------------------------------------------------------------------------------------------
def _decisions(st, kmax):
    return [d for d in st["decisions"] if d[1] <= kmax]


def check_decisions(ref, ex, ks, what):
    kmax = max(ks)
    want, exact = _decisions(ref[kmax], kmax), _decisions(ex[kmax], kmax)
    if want != exact:
        pytest.fail(f"{what}: the restatement and its exact evaluation decide differently up to k = {kmax} "
                    f"({want} against {exact}): the case says nothing about the kernels, fix the case")


def check_state(method, k, got, want, exact, what):
    """One solve stopped at k against the restatement's state; returns the largest (err / spread ratio, where)."""
    what = f"{what} k={k}"
    L = want["x"].shape[0]
    assert got["ret"] == want["ret"], (what, "return value", got["ret"], want["ret"])
    assert got["iters"] == want["iters"], (what, "iters", got["iters"], want["iters"])
    assert got["hist"].size == want["hist"].size, (what, "history length", got["hist"].size, want["hist"].size)
    assert got["seed"] == want["seed"], (what, "seed", got["seed"], want["seed"])
    assert np.array_equal(got["stop"], want["stop_iter"]), (what, "stop iterations", got["stop"], want["stop_iter"])
    ratio = _hold(f"{what} r", got["r"], want["r"], exact["r"])
    for j in range(L):
        ratio = max(ratio, _hold(f"{what} x[{j}] (pi {want['shift']['pi'][j]:.6g}, zeta {want['shift']['zeta'][j]:.6g})",
                                 got["x"][j], want["x"][j], exact["x"][j]))
    hspread = max(_rel(exact["hist"][i], want["hist"][i]) for i in range(want["hist"].size))
    for i in range(1, want["hist"].size):
        ratio = max(ratio, _hold(f"{what} hist[{i}]", got["hist"][i], want["hist"][i], exact["hist"][i], hspread))
    return ratio


def solve_k(B, dm, method, k, sigma, seed, b, tol, x0=None):
    """One solve with shift_max_iter = k on host vectors from x0 (a numpy (L, n) initial x_set; None: zero), or in place on x0
    if it is a CUDA tensor."""
    L, n = sigma.size, b.size
    B.set_options(shift_tol=tol, shift_max_iter=k)
    if x0 is None or isinstance(x0, np.ndarray):
        x, r = np.zeros((L, n)) if x0 is None else x0.copy(), b.copy()
        ret, st = dm.shifted_solve(method, x, r, sigma, seed)
    else:
        import torch
        x, rt = x0, torch.from_numpy(b.copy()).cuda()
        ret, st = dm.shifted_solve(method, x, rt, sigma, seed)
        x, r = x.cpu().numpy(), rt.cpu().numpy()
    seed_out, stop = B.last_shift_info(L)
    assert st["iters"] == B.last_history().size - 1, (st["iters"], B.last_history().size)
    return dict(ret=ret, iters=st["iters"], x=x, r=r, hist=B.last_history(), seed=seed_out, stop=stop)


def _device_x_set(x0, offset):
    """x0 (L, n) as a CUDA tensor: contiguous, or a view one element into a larger tensor (every row misaligned for even n)."""
    import torch
    t = torch.from_numpy(x0).cuda()
    if not offset:
        return t
    big = torch.zeros(x0.size + 1, dtype=torch.float64, device="cuda")
    big[1:].view(x0.shape).copy_(t)
    return big[1:].view(x0.shape)


def check_stopped_shifts(method, outs, what):
    """A shift that has stopped does not move: its x_j at every later k is its x_j at the first k past its stop."""
    if method in LOP:
        return
    ks = sorted(outs)
    last = outs[ks[-1]]
    for j, s in enumerate(last["stop"]):
        if s == 0 or (method == FIXED and j == last["seed"]):    # shifted_lopbicg's seed keeps iterating after it stopped
            continue
        after = [k for k in ks if k >= s and outs[k]["stop"][j] == s]
        for k in after[1:]:
            assert outs[k]["x"][j].tobytes() == outs[after[0]]["x"][j].tobytes(), (what, "stopped shift moved", j, s, after[0], k)


def run_states(B, O, spec, method, L, scale, seed, tol=1e-12, ks=KS, label=None, keep_p=True, x0=False, device=None):
    """Solve for every k in ks on one handle, hold each state to the restatement.  x0: start from helpers.initial_x_set instead
    of zero; device: solve in place on a CUDA tensor, "aligned" or at a one-element "offset".  Returns {k: the solve's results}."""
    label = label or f"{spec} {method} L={L} seed={seed} tol={tol:g}"
    label += (" x0" if x0 else "") + (f" device-{device}" if device else "")
    n, ptr, col, val = _matrix(B, spec)
    sigma, b = _problem(O, n, ptr, col, val, L, scale, seed)
    ref, ex = reference(B, O, spec, method, L, scale, seed, tol, ks, keep_p, x0)
    xs = initial_x_set(L, n) if x0 else np.zeros((L, n))
    check_decisions(ref, ex, ks, label)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    worst, outs = (0.0, ""), {}
    try:
        for k in ks:
            start = xs if device is None else _device_x_set(xs, device == "offset")
            outs[k] = solve_k(B, dm, method, k, sigma, seed, b, tol, start)
            worst = max(worst, check_state(method, k, outs[k], ref[k], ex[k], label))
    finally:
        dm.destroy()
    check_stopped_shifts(method, outs, label)
    print(f"[shifted-state] {label}: largest err/spread ratio {worst[0]:.3g} ({worst[1]})")
    return outs


# ---- the shifted cases --------------------------------------------------------------------------------------------
# (id, matrix, L, shift scale, seed, tol): every SHIFTED_LOP_CASES entry and the fixed-seed extras (L = 1, seeds 2 and 4 of 5),
# then the switch cases and test_shifted.c's set-up with tol = 1e-6, where shifts stop and the seed switches within 17 iterations
CASES = ([(c[0], c[1:4], c[4], c[5], c[6], c[7]) for c in FIXED_CASES] +
         [(f"{c[0]}_tol1e-6", c[1:4], c[4], c[5], c[6], 1e-6) for c in FIXED_CASES
          if c[0] in ("sh_convdiff_g40_L6_switch", "sh_stencil15_g12_L4_switch", "sh_test_shifted_stencil15_g12")])


# The last k at which a case's own rounding spread stays under MAX_SPREAD, (other methods, PIPE-LOP), where that is before
# k = 17: as the residual falls its spread grows, fastest under the pipelined recurrences of PIPE-LOP.  States past it say
# nothing about the kernels, so they are not compared.  Both sides of the batch boundary (k = 8, 9) stay in every case but
# the PIPE-LOP ones marked 3 or 7.
KMAX = {"sh_convdiff_g40_L6_switch": (15, 3), "sh_convdiff_g40_L6_switch_tol1e-6": (11, 3), "sh_stencil15_g12_L4_switch": (13, 7),
        "sh_stencil15_g12_L4_switch_tol1e-6": (17, 7), "small_n17": (17, 7), "table_edges": (9, 7)}


def kmax(name, method):
    other, pipe = KMAX.get(name, (17, 9))
    return pipe if method == "shifted_pipe_lopbicgstab" else other


def _ks(B, O, case, method=None):
    _, spec, L, scale, seed, tol = case
    ks_ = switch_iteration(B, O, spec, L, scale, seed, tol)
    ks = sorted(set(KS) | ({ks_ - 1, ks_, ks_ + 1, ks_ + 2} if ks_ else set()))
    return tuple(k for k in ks if method is None or k <= kmax(case[0], method))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_shifted_cases_state(B, O, case, method):
    _, spec, L, scale, seed, tol = case
    ks = _ks(B, O, case, method)
    outs = run_states(B, O, spec, method, L, scale, seed, tol, ks, label=f"{case[0]} {method}")
    if method == SWITCHING and case[0].endswith("switch_tol1e-6"):
        ks_ = switch_iteration(B, O, spec, L, scale, seed, tol)
        assert outs[ks_]["seed"] != seed and outs[ks_ - 1]["seed"] == seed        # the solve that ends on the switch


def test_device_path_every_k(B, O):
    """bicg_shifted_solve_dev, on an aligned tensor and on a view at a one-element offset, leaves the host path's bits after
    every k, through both seed switches and the stops of the tol = 1e-6 cases."""
    import torch
    for case in [c for c in CASES if c[0].endswith("_tol1e-6")]:
        _, spec, L, scale, seed, tol = case
        n, ptr, col, val = _matrix(B, spec)
        sigma, b = _problem(O, n, ptr, col, val, L, scale, seed)
        dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
        try:
            for method in METHODS:
                for k in _ks(B, O, case):
                    host = solve_k(B, dm, method, k, sigma, seed, b, tol)
                    big = torch.zeros(L * n + 1, dtype=torch.float64, device="cuda")
                    for xt in (torch.zeros((L, n), dtype=torch.float64, device="cuda"), big[1:].view(L, n)):
                        dev = solve_k(B, dm, method, k, sigma, seed, b, tol, x0=xt)
                        for key in ("ret", "iters", "seed"):
                            assert dev[key] == host[key], (case[0], method, k, key)
                        assert np.array_equal(dev["stop"], host["stop"]), (case[0], method, k)
                        for key in ("x", "r", "hist"):
                            assert dev[key].tobytes() == host[key].tobytes(), (case[0], method, k, key, xt.data_ptr() % 16)
        finally:
            dm.destroy()


# ---- row counts and shift counts --------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", ["small_n17", "small_n2111", "ragged_4001"])
def test_row_counts_state(B, O, name, method):
    """n = 17 and 2111 (odd: the one-row tail of the two-rows-per-thread update loops) and a ragged matrix whose rows often
    hold only their diagonal; 5 shifts around a middle seed."""
    assert name in MATRICES
    run_states(B, O, name, method, 5, 0.05, 2, ks=tuple(k for k in KS if k <= kmax(name, method)))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("L", [1, 2, 33, 512, 513])
def test_shift_counts_state(B, O, L, method):
    """No shift besides the seed, one, more than a warp, as many as and more than the 512 threads of the scalar kernels."""
    run_states(B, O, ("stencil15", 12, 14.0), method, L, 0.01 / L if L > 1 else 0.01, L - 1 if L % 2 else L // 2)


# shift counts at which the coefficient table of the update kernel needs a second pass: sh_vec_shift keeps 52 B per active
# shift (945 fit into 48 KB), lop_vec_update 48 B per non-seed shift next to its 2640 B of static shared memory (969 fit)
EDGES = ([(m, L) for m in (SWITCHING, FIXED) for L in (945, 946, 4470, 4471, 8192)] +
         [(m, L) for m in LOP for L in (970, 971, 1025, 1026, 4788, 4789, 8192)])


@pytest.mark.parametrize("method,L", EDGES, ids=[f"{m}-L{L}" for m, L in EDGES])
def test_table_edges_state(B, O, method, L):
    """Both sides of the shared-memory edges of the update kernels' coefficient tables, with the seed in the middle: shifts
    on either side of it, in the first pass and in later ones."""
    run_states(B, O, "small_n17", method, L, 0.5 / L, L // 2, ks=tuple(k for k in KS if k <= kmax("table_edges", method)))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", STANDALONE, ids=[c[0] for c in STANDALONE])
def test_standalone_spmv_state(B, O, case, method):
    """Every forced stand-alone SpMV variant: the shifted epilogue fma(sigma, x[row], acc) under the epilogues with no, one
    and two dots that the shifted drivers use."""
    _, name, opts, _, _ = case
    B.set_options(**opts)
    run_states(B, O, name, method, 5, 0.2, 2, ks=(1, 2, 3), label=f"{case[0]} {method}")


@pytest.mark.parametrize("method", METHODS)
def test_large_matrix_every_shift_state(B, O, method):
    """216 k rows (T', g = 60), 64 shifts: every x_j at a realistic size."""
    run_states(B, O, "stencil15_g60", method, 64, 0.5 / 64, 0, ks=(1, 2, 3), keep_p=False)


# ---- any number of shifts ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
def test_many_shifts_match_512(B, O, method):
    """With tol = 0 and shift_max_iter = k no shift stops and the seed never switches, so every shift's x_j depends only on
    the seed and its own sigma: the first 512 shifts of an 8192- and a 1000-shift solve (several passes of the coefficient
    table) are those of a 512-shift solve, bit for bit.  Solved to convergence, every one of the 8192 shifts has a relative
    residual <= 1e-10."""
    n, ptr, col, val = _matrix(B, ("stencil15", 12, 14.0))
    sigma = (np.arange(8192) + 1) * (0.01 / 512)
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[0], np.ones(n), b)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        for k in (3, 9):
            base = solve_k(B, dm, method, k, sigma[:512], 0, b, 0.0)
            for L in (1000, 8192):
                many = solve_k(B, dm, method, k, sigma[:L], 0, b, 0.0)
                assert many["ret"] == base["ret"] and many["hist"].tobytes() == base["hist"].tobytes(), (method, k, L)
                assert many["r"].tobytes() == base["r"].tobytes(), (method, k, L)
                for j in range(512):
                    assert many["x"][j].tobytes() == base["x"][j].tobytes(), (method, k, L, j)
        B.set_options(shift_tol=1e-12, shift_max_iter=1000)
        x, r = np.zeros((8192, n)), b.copy()
        ret, st = dm.shifted_solve(method, x, r, sigma, 0)
        assert st["converged"], (method, ret)
        res = dm.shift_residuals(x, b, sigma)
        assert res.max() <= 1e-10, (method, int(res.argmax()), res.max())
    finally:
        dm.destroy()


# ---- nonzero initial x_set ------------------------------------------------------------------------------------------------
# None of the four solvers forms b - A x0: they add corrections to each x_j, so x_j = x0_j + correction.  x0 = 0.1 standard
# normal keeps |x0| no larger than the corrections, which set max|x_j| in the max-norm rule: a large x0 would hide their error.
X0_CASES = [c for c in CASES if c[0] in ("sh_convdiff_g40_L6_switch", "fx_stencil15_g12_L5_seed2")] + [
    ("small_n17", "small_n17", 5, 0.05, 2, 1e-12)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", X0_CASES, ids=[c[0] for c in X0_CASES])
def test_nonzero_x0_state(B, O, case, method):
    _, spec, L, scale, seed, tol = case
    run_states(B, O, spec, method, L, scale, seed, tol, _ks(B, O, case, method), label=f"{case[0]} {method}", x0=True)


X0_EDGES = [(m, L) for m, L in EDGES if L in (945, 946, 970, 971)]


@pytest.mark.parametrize("method,L", X0_EDGES, ids=[f"{m}-L{L}" for m, L in X0_EDGES])
def test_nonzero_x0_table_edges_state(B, O, method, L):
    """The update kernels' coefficient tables in one pass and in two, adding to a nonzero x_j on either side of the seed."""
    run_states(B, O, "small_n17", method, L, 0.5 / L, L // 2, ks=tuple(k for k in KS if k <= kmax("table_edges", method)), x0=True)


@pytest.mark.parametrize("device", ["aligned", "offset"])
@pytest.mark.parametrize("method", METHODS)
def test_nonzero_x0_device_path_state(B, O, method, device):
    """bicg_shifted_solve_dev in place on the caller's nonzero x_set, through the seed switch: held to the restatement itself,
    not only to the host path."""
    case = next(c for c in X0_CASES if c[0] == "sh_convdiff_g40_L6_switch")
    _, spec, L, scale, seed, tol = case
    run_states(B, O, spec, method, L, scale, seed, tol, _ks(B, O, case, method), label=f"{case[0]} {method}", x0=True, device=device)
