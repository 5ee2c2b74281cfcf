"""GPU: the shifted solvers on device-resident vectors (bicg_shifted_solve_dev, DeviceMatrix.shifted_solve with CUDA tensors) and
DeviceMatrix.solve with CUDA tensors (bicg_solve, device_vectors = 1), from zero and from nonzero initial guesses.

For each of the four shifted methods the same problem runs through the host path (numpy) and the device path (tensors updated in
place), with BICG_SHIFT_ERROR=1 and rank 0's printout on.  These must be bitwise equal: x_set, r, the return value,
bicg_last_history, bicg_last_shift_info, iters / converged / final_res, kernel_launches, the BICG_SHIFT_ERROR errors and the
stdout apart from the Total time / Avg time/iter values.  The device path must leave the tensors where they were (data_ptr),
report h2d_bytes = d2h_bytes = 0, and shift_residuals on the returned tensor must equal the in-solver report.  Cases: the shifted
cases (seed-switching ones included) and the fixed-seed extras, n = 17 and n = 3001 with L in {1, 5, 64, 513}, and x_set as a
view at a one-element offset into a larger tensor (every block misaligned for even n; odd n misaligns every other block)."""
import ctypes as C
import re

import numpy as np
import pytest

from helpers import SMALL_CASES, RR, global_csr, initial_guess
from shifted_fixed_cases import FIXED_CASES
from shifted_lop_cases import SHIFTED_LOP_CASES, shifted_lop_problem

pytestmark = pytest.mark.gpu
METHODS = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]
PLAIN = ["bicgstab", "ca_bicgstab", "pipe_bicgstab", "pipe_bicgstab_rr"]
CASES = SHIFTED_LOP_CASES + [c[:7] for c in FIXED_CASES[len(SHIFTED_LOP_CASES):]]
SIZES = [("random", 17, 5), ("random", 3001, 8)]
_MASK = re.compile(r"(Total time   :|Avg time/iter:) \S+")


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _flush_out(B, capfd):
    B.lib.bicg_synchronize()
    C.CDLL(None).fflush(None)
    return capfd.readouterr().out


def _after(B, L, capfd):
    seed, stop = B.last_shift_info(L)
    return dict(out=_MASK.sub(r"\1", _flush_out(B, capfd)), hist=B.last_history(), seed=seed, stop=stop, err=B.last_shift_error(L))


def _host_and_device(B, dm, method, x0, b, sigma, seed, capfd, offset=False, torch_sigma=False):
    """Run the problem through both paths; returns (host results, device results, device x_set / r as numpy)."""
    import torch
    L, n = sigma.size, b.size
    B.set_options(shift_error=1)
    capfd.readouterr()
    x = x0.copy(); r = b.copy()
    k, st = dm.shifted_solve(method, x, r, sigma, seed)
    host = dict(k=k, st=st, x=x, r=r, **_after(B, L, capfd))
    if offset:                      # x_set at a one-element offset inside a larger tensor, with sentinels on either side
        big = torch.full((L * n + 2,), 7.0, dtype=torch.float64, device="cuda")
        xt = big[1:1 + L * n].view(L, n)
        xt.copy_(torch.from_numpy(x0))
        assert xt.data_ptr() % 16 == 8
    else:
        xt = torch.from_numpy(x0.copy()).cuda()
    rt = torch.from_numpy(b.copy()).cuda()
    ptrs = (xt.data_ptr(), rt.data_ptr())
    k, st = dm.shifted_solve(method, xt, rt, torch.from_numpy(sigma) if torch_sigma else sigma, seed)
    dev = dict(k=k, st=st, **_after(B, L, capfd))
    B.set_options(shift_error=0)
    assert (xt.data_ptr(), rt.data_ptr()) == ptrs
    if offset:
        assert big[0].item() == 7.0 and big[-1].item() == 7.0        # nothing written outside x_set
    dev["x"], dev["r"] = xt.cpu().numpy(), rt.cpu().numpy()
    # the check of the returned tensor is the in-solver report, bit for bit
    res = dm.shift_residuals(xt, torch.from_numpy(b).cuda(), sigma)
    assert _bits(res) == _bits(dev["err"]), (method, res, dev["err"])
    return host, dev


def _assert_same(host, dev, what):
    assert dev["k"] == host["k"], what
    for key in ("x", "r", "hist", "err"):
        assert _bits(dev[key]) == _bits(host[key]), (what, key)
    assert dev["seed"] == host["seed"] and np.array_equal(dev["stop"], host["stop"]), what
    for key in ("iters", "converged", "kernel_launches"):
        assert dev["st"][key] == host["st"][key], (what, key)
    assert _bits(dev["st"]["final_res"]) == _bits(host["st"]["final_res"]), what
    assert dev["out"] == host["out"], what
    assert dev["st"]["h2d_bytes"] == 0 and dev["st"]["d2h_bytes"] == 0, what
    assert host["st"]["h2d_bytes"] > 0, what
    assert host["err"].size == host["x"].shape[0], what


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_device_path_matches_host_path(B, O, capfd, method, case):
    B.set_options(quiet=0, shift_tol=1e-12, shift_max_iter=1000)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    dm = B.DeviceMatrix(blk)
    host, dev = _host_and_device(B, dm, method, np.zeros((sigma.size, n)), b, sigma, seed, capfd)
    dm.destroy()
    B.set_options(quiet=1)
    _assert_same(host, dev, (method, case[0]))
    if case[0] == "sh_convdiff_g40_L6_switch" and method == "shifted_lopbicg_switching":
        assert host["seed"] != seed and "k: " in host["out"]          # the seed does switch, and its lines are compared


@pytest.mark.parametrize("L", [1, 5, 64, 513])
@pytest.mark.parametrize("mat", SIZES, ids=[f"{k}{g}" for k, g, _ in SIZES])
@pytest.mark.parametrize("method", METHODS)
def test_device_path_matches_host_path_sizes(B, O, capfd, method, mat, L):
    """n = 17 and n = 3001 (odd: every other block of a device x_set is misaligned), nonzero initial guesses."""
    B.set_options(quiet=0, shift_tol=1e-12, shift_max_iter=1000)
    blk, n, ptr, col, val = global_csr(B, *mat)
    seed = L // 2
    sigma = (np.arange(L) + 1) * (0.05 / L)
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[seed], np.ones(n), b)
    x0 = np.random.default_rng(L + n).uniform(-1e-3, 1e-3, (L, n))
    dm = B.DeviceMatrix(blk)
    host, dev = _host_and_device(B, dm, method, x0, b, sigma, seed, capfd, torch_sigma=L == 5)
    dm.destroy()
    B.set_options(quiet=1)
    _assert_same(host, dev, (method, mat, L))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", [SHIFTED_LOP_CASES[0], SHIFTED_LOP_CASES[1], SHIFTED_LOP_CASES[3]], ids=lambda c: c[0])
def test_misaligned_view(B, O, capfd, method, case):
    """x_set as a view at a one-element offset into a larger tensor: with even n (stencil15 g12, convdiff g40) every block starts
    8 bytes past a 16-byte boundary, with odd n (laplace5 g37) every other one; the results are still the host path's bits."""
    B.set_options(quiet=0, shift_tol=1e-12, shift_max_iter=1000)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    dm = B.DeviceMatrix(blk)
    host, dev = _host_and_device(B, dm, method, np.zeros((sigma.size, n)), b, sigma, seed, capfd, offset=True, torch_sigma=True)
    dm.destroy()
    B.set_options(quiet=1)
    _assert_same(host, dev, (method, case[0], "offset"))


@pytest.mark.parametrize("method", PLAIN)
@pytest.mark.parametrize("case", [SMALL_CASES[0], SMALL_CASES[3]], ids=lambda c: c[0])
def test_plain_solve_tensors_match_numpy(B, O, method, case):
    """From x0 = 0 and from a nonzero x0 (r0 = b - A x0 then differs from b): the tensor path is the numpy path, bit for bit."""
    import torch
    B.set_options(quiet=1, tol=1e-10, max_iter=1000)
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    b = O.spmv(n, ptr, col, val, np.ones(n))
    kw = RR if method == "pipe_bicgstab_rr" else {}
    dm = B.DeviceMatrix(blk)
    try:
        for x0 in (np.zeros(n), initial_guess("normal", n)):
            x = x0.copy(); r = b.copy()
            it_h, st_h = dm.solve(method, x, r, **kw)
            hist_h = B.last_history()
            xt = torch.from_numpy(x0.copy()).cuda(); rt = torch.from_numpy(b.copy()).cuda()
            ptrs = (xt.data_ptr(), rt.data_ptr())
            it_d, st_d = dm.solve(method, xt, rt, **kw)
            hist_d = B.last_history()
            assert (xt.data_ptr(), rt.data_ptr()) == ptrs
            assert it_d == it_h and st_d["iters"] == st_h["iters"] and st_d["converged"] == st_h["converged"]
            assert _bits(st_d["final_res"]) == _bits(st_h["final_res"])
            assert _bits(xt.cpu().numpy()) == _bits(x) and _bits(rt.cpu().numpy()) == _bits(r) and _bits(hist_d) == _bits(hist_h)
            assert st_d["h2d_bytes"] == 0 and st_d["d2h_bytes"] == 0
            assert np.abs(x - 1.0).max() < 1e-6
    finally:
        dm.destroy()
