"""GPU: the batched multiply y_j = alpha (A + sigma_j I) x_j + beta y_j on a resident matrix (bicg_matrix_multiply, _async).  Its
row sums are bicg_spmv's, whatever batch a vector runs in, and its epilogue is pinned down in include/bicgstab_b200.h, so every
result is checked bit for bit: against spmv, against a correctly rounded epilogue, across batch sizes, against the synchronous
sequence when stream-ordered or replayed from a CUDA graph.  The cases cover both SpMV plan kinds (the TMA tile kernel for
stencil15 and laplace5, the row-split kernel for random_k32 and the chunked matrix) and several lanes settings."""
import numpy as np
import pytest

from helpers import initial_x_set
from rowsum_model import fma as _fma
from test_gpu_set_values import _case_block, _perturbed, _values

pytestmark = pytest.mark.gpu

CASES = ["stencil15", "laplace5", "random_k32", "chunked"]
NV_MAX = 8                                      # vectors per launch (MUL_NV_MAX of csrc/spmv.cuh)
NVECS = [1, 3, NV_MAX, NV_MAX + 1, 17]          # full, partial and several launches


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, tol=1e-10, max_iter=400, mega=1, resident=0, spmv_lanes=0)
    yield
    B.set_options(tol=1e-15, max_iter=1000, mega=1, resident=1, spmv_lanes=0)


def _torch():
    import torch
    return torch


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _xs(nvec, n, seed):
    return np.random.default_rng(seed + 31 * nvec).standard_normal((nvec, n))


@pytest.fixture(scope="module", params=CASES)
def case(request, B):
    B.set_options(quiet=1, cache=1)
    blk = _case_block(B, request.param)
    dm = B.DeviceMatrix(blk)
    yield request.param, blk, dm
    dm.destroy()


def test_matches_spmv(B, case):
    """alpha = 1, beta = 0, no sigma: every y_j equals spmv(x_j) bit for bit -- synchronous from host and device vectors, and
    stream-ordered -- for full, partial and several launches."""
    torch = _torch()
    name, blk, dm = case
    n = blk.n_loc
    for nvec in NVECS:
        x = _xs(nvec, n, 1)
        want = [_bits(dm.spmv(x[j])) for j in range(nvec)]
        y_host = dm.multiply(x)
        tx = torch.from_numpy(x).cuda()
        y_dev = dm.multiply(tx)
        y_async = torch.full((nvec, n), np.nan, dtype=torch.float64, device="cuda")
        dm.multiply_async(tx, y_async)
        torch.cuda.synchronize()
        for j in range(nvec):
            assert _bits(y_host[j]) == want[j], (name, nvec, j, "host")
            assert _bits(y_dev[j]) == want[j], (name, nvec, j, "device")
            assert _bits(y_async[j]) == want[j], (name, nvec, j, "async")
    # one vector of shape (n_loc,)
    x1 = _xs(1, n, 2)[0]
    assert _bits(dm.multiply(x1)) == _bits(dm.spmv(x1))


def test_epilogue_is_correctly_rounded(B, case):
    """Random x, y, alpha, beta, sigma (some sigma_j = 0, beta = 0 with y full of NaN, negative alpha): y equals the header's
    epilogue on spmv's row sums -- t = fma(sigma_j, x_j, rowsum), then alpha t or fma(alpha, t, beta y) -- bit for bit."""
    torch = _torch()
    name, blk, dm = case
    n = blk.n_loc                                  # every row
    nvec = 3
    rng = np.random.default_rng(11)
    x = rng.standard_normal((nvec, blk.n_loc))
    rowsum = np.stack([dm.spmv(x[j]) for j in range(nvec)])
    for alpha, beta, sigma in [(1.5, 0.0, None), (-0.75, 0.0, np.array([0.0, 0.3, -1.25])), (-1.0, 1.0, np.array([2.0, 0.0, 0.0])),
                               (0.625, -2.5, np.array([0.1, -0.7, 0.0])), (-3.0, 0.5, None)]:
        y0 = np.full((nvec, blk.n_loc), np.nan) if beta == 0.0 else rng.standard_normal((nvec, blk.n_loc))
        t = rowsum[:, :n] if sigma is None else _fma(sigma[:, None], x[:, :n], rowsum[:, :n])
        want = alpha * t if beta == 0.0 else _fma(alpha, t, beta * y0[:, :n])
        got_host = dm.multiply(x, y0.copy(), alpha=alpha, beta=beta, sigma=sigma)
        ty = torch.from_numpy(y0).cuda()
        dm.multiply_async(torch.from_numpy(x).cuda(), ty, alpha=alpha, beta=beta,
                          sigma=None if sigma is None else torch.from_numpy(sigma).cuda())
        torch.cuda.synchronize()
        for got in (got_host, ty.cpu().numpy()):
            assert not np.isnan(got).any(), (name, alpha, beta)
            assert _bits(got[:, :n]) == _bits(want), (name, alpha, beta, sigma)
            assert _bits(got) == _bits(got_host), (name, alpha, beta, sigma)


def test_batch_independence(B, case):
    """y_j of one nvec = 17 call equals y_j of 17 single-vector calls, with a shift and beta != 0."""
    torch = _torch()
    name, blk, dm = case
    n, nvec = blk.n_loc, 17
    x = torch.from_numpy(_xs(nvec, n, 3)).cuda()
    y0 = torch.from_numpy(_xs(nvec, n, 4)).cuda()
    sigma = torch.from_numpy(np.linspace(-1.0, 2.0, nvec)).cuda()
    y = y0.clone()
    dm.multiply_async(x, y, alpha=-0.5, beta=2.0, sigma=sigma)
    singles = y0.clone()
    for j in range(nvec):
        dm.multiply_async(x[j], singles[j], alpha=-0.5, beta=2.0, sigma=sigma[j:j + 1])
    torch.cuda.synchronize()
    assert _bits(y) == _bits(singles), name


def test_against_oracle(B, O, case):
    name, blk, dm = case
    ptr, col, val = B.block_to_global_csr(blk)
    x = _xs(5, blk.n_loc, 5)
    y = dm.multiply(x)
    for j in range(5):
        y_ref = O.spmv(blk.n, ptr, col, val, x[j], long_double=True)
        assert np.abs(y[j] - y_ref).max() <= 1e-13 * np.abs(y_ref).max(), (name, j)


# ---- stream order, capture, shifted solutions (stencil15: the TMA tile kernel and the persistent solver) ----------------------
METHOD = "bicgstab"
# The solve stops on its recursive residual sqrt(dot_r / dot_zero) <= tol.  The true residual ||b - A x|| / ||b|| differs from
# it by the rounding the recursion accumulates, O(iterations * eps * ||A|| ||x|| / ||b||): about 1e-13 for these well
# conditioned diagonally dominant matrices, so a gap of tol / 10 is generous and still says the two agree.
TOL = 1e-10
RES_GAP = TOL / 10


def _sync_sequence(B, dm, vals, ones):
    """set_values -> b = A 1 -> solve from x = 0 -> r = b - A x, synchronously"""
    dm.set_values(vals)
    b = dm.multiply(ones)
    x, r = np.zeros_like(b), b.copy()
    it, st = dm.solve(METHOD, x, r)
    res = dm.multiply(x, b.copy(), alpha=-1.0, beta=1.0)
    return dict(b=_bits(b), x=_bits(x), r=_bits(r), res=_bits(res), it=it), np.linalg.norm(res) / np.linalg.norm(b), st["final_res"]


class _Async:
    """The same sequence enqueued on one stream: set_values_async, multiply_async, solve_async, multiply_async"""

    def __init__(self, B, dm, n):
        torch = _torch()
        self.dm = dm
        f = lambda: torch.empty(n, dtype=torch.float64, device="cuda")
        self.vals = torch.empty(int(dm.blk.diag.nz), dtype=torch.float64, device="cuda")
        self.ones, self.b, self.x, self.r, self.res = f(), f(), f(), f(), f()
        self.result = torch.zeros(24, dtype=torch.uint8, device="cuda")

    def enqueue(self):
        dm = self.dm
        dm.set_values_async(self.vals)
        dm.multiply_async(self.ones, self.b)
        self.x.zero_()
        self.r.copy_(self.b)
        dm.solve_async(METHOD, self.x, self.r, result=self.result)
        self.res.copy_(self.b)
        dm.multiply_async(self.x, self.res, alpha=-1.0, beta=1.0)

    def got(self, B):
        rec = B.decode_result(self.result)
        return dict(b=_bits(self.b), x=_bits(self.x), r=_bits(self.r), res=_bits(self.res), it=rec["iters"])


@pytest.mark.parametrize("mega", [0, 1])
def test_stream_order_without_host_synchronisation(B, mega):
    """update values, form b = A 1, solve, true residual b - A x: all on a side stream with no host synchronisation between
    them, bit-identical to the synchronous sequence; ||b - A x|| / ||b|| agrees with the solve's final residual."""
    torch = _torch()
    B.set_options(mega=mega, tol=TOL)
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    dv, _ = _values(blk)
    vals = _perturbed(dv, 2)
    ones = np.ones(n)
    dm = B.DeviceMatrix(blk)
    try:
        want, true_res, final_res = _sync_sequence(B, dm, vals, ones)
        assert abs(true_res - final_res) <= RES_GAP and final_res <= TOL, (true_res, final_res)
        dm.set_values(dv)                                    # back to the creation's values
        dm.prepare_async(METHOD)
        a = _Async(B, dm, n)
        a.vals.copy_(torch.from_numpy(vals))
        a.ones.copy_(torch.from_numpy(ones))
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            a.enqueue()
        s.synchronize()
        assert a.got(B) == want
    finally:
        dm.destroy()


def test_captured_sequence_replay(B):
    """The sequence captured in torch.cuda.graph, replayed with new values and a new x in the same buffers: every replay equals
    an uncaptured run of the same sequence bit for bit."""
    torch = _torch()
    B.set_options(tol=TOL)
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    dv, _ = _values(blk)
    dm = B.DeviceMatrix(blk)
    try:
        dm.prepare_async(METHOD)
        a = _Async(B, dm, n)
        a.vals.copy_(torch.from_numpy(dv))
        a.ones.fill_(1.0)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            a.enqueue()
        for k in (2, 3, 4):
            vals, xin = _perturbed(dv, k), 1.0 + 0.01 * _xs(1, n, k)[0]
            a.vals.copy_(torch.from_numpy(vals))
            a.ones.copy_(torch.from_numpy(xin))
            g.replay()
            torch.cuda.synchronize()
            got = a.got(B)
            a.enqueue()                                      # uncaptured, same inputs
            torch.cuda.synchronize()
            assert got == a.got(B), k
            want, _, _ = _sync_sequence(B, dm, vals, xin)
            assert got == want, k
        del g
    finally:
        dm.destroy()


def test_shifted_solution_residuals(B):
    """After a shifted solve, multiply(x_set, y = b per shift, alpha = -1, beta = 1, sigma) gives b - (A + sigma_j I) x_j; its
    norms over ||b|| agree with shift_residuals to 1e-12 relative (the components are the same, only the norms' summation
    orders differ; one lane per row, as shift_residuals sums a row)."""
    B.set_options(spmv_lanes=1, shift_tol=1e-12, shift_max_iter=1000)
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    dm = B.DeviceMatrix(blk)
    try:
        sigma = np.array([0.0, 0.5, 1.5, 3.0])
        b = dm.spmv(np.ones(n))
        xs = initial_x_set(sigma.size, n)
        dm.shifted_solve("shifted_lopbicgstab", xs, b.copy(), sigma, 0)
        res = dm.multiply(xs, np.ascontiguousarray(np.tile(b, (sigma.size, 1))), alpha=-1.0, beta=1.0, sigma=sigma)
        got = np.linalg.norm(res, axis=1) / np.linalg.norm(b)
        want = dm.shift_residuals(xs, b, sigma)
        assert np.all(np.abs(got - want) <= 1e-12 * want), (got, want)
    finally:
        dm.destroy()
