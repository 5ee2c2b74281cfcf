"""GPU: new values on a resident matrix (bicg_matrix_set_values, _async, bicg_matrix_shift_diagonal).  An update rewrites the
merged values and rebuilds the persistent kernel's value tables and packed values with the pass bicg_matrix_create runs, and keeps
everything else on the handle.  So every result after an update must be bit for bit that of a handle freshly created, in the same
process, from blocks holding the same values: x, r, history, iterations and which CTAs ran resident, coded and packed, on every
loop path (persistent kernel resident and streaming, kernel-per-phase), for the plain and the shifted solvers, synchronous,
stream-ordered and captured into a CUDA graph."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import METHODS, RR, initial_guess, initial_x_set

pytestmark = pytest.mark.gpu

SHIFTED = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]
CASES = ["stencil15", "laplace5", "random_k32", "chunked", "resident"]
VARIANTS = ["default", "columns32", "values8"]


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, tol=1e-10, max_iter=400, mega=1, resident=0, mega_lanes=0, shift_tol=1e-12,
                  shift_max_iter=1000, shift_error=0)
    yield
    B.set_options(tol=1e-15, max_iter=1000, mega=1, resident=1, mega_lanes=0)


def _torch():
    import torch
    return torch


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


_CHUNKED = []


def _chunked_matrix():
    """Rows of ~10 entries plus three dense rows, longer than a stage: the persistent kernel's plan cuts them into chunk tiles."""
    if not _CHUNKED:
        n = 40000
        rng = np.random.default_rng(5)
        rows = np.repeat(np.arange(n), 10)
        cols = rng.integers(0, n, size=rows.size)
        A = sp.csr_matrix((-(0.5 + 0.5 * rng.random(rows.size)), (rows, cols)), shape=(n, n))
        A = sp.lil_matrix(A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 1.0))
        for r in (0, 20011, n - 1):
            A[r, :] = -2.0 / n
            A[r, r] = 4.0
        A = sp.csr_matrix(A)
        A.sort_indices()
        _CHUNKED.append(A)
    return _CHUNKED[0]


def _case_block(B, case):
    if case == "chunked":
        A = _chunked_matrix()
        return B.blocks_from_csr(A.shape[0], A.indptr, A.indices, A.data)
    kind, g, p0 = {"stencil15": ("stencil15", 24, 14.0), "laplace5": ("laplace5", 60, 0.0), "random_k32": ("random", 3001, 32),
                   "resident": ("stencil15", 12, 14.0)}[case]
    return B.gen_block(kind, g, p0)


def _values(blk):
    return blk.diag_arrays()[0].copy(), blk.offd_arrays()[0].copy()


def _with_values(blk, dv, ov):
    """blk with its values overwritten in place (the pattern stays): what a fresh handle is created from."""
    blk.diag_arrays()[0][:] = dv
    if ov.size:
        blk.offd_arrays()[0][:] = ov
    return blk


def _perturbed(v, k):
    """Value set k: every value scaled by one of 1, 1 + 1/64, ..., 1 + 6/64 in a pattern that depends on k."""
    return v * (1.0 + ((np.arange(v.size) * (2 * k + 1) + k) % 7) / 64.0)


def _src(src, dv, ov):
    """The values as numpy arrays or as CUDA tensors; offd None when the block has no offd entries."""
    if src == "torch":
        torch = _torch()
        dv, ov = torch.from_numpy(dv).cuda(), torch.from_numpy(ov).cuda()
    return dv, (ov if ov.shape[0] else None)


def _run(B, dm, method, b, x0, variant="default"):
    dm.stream_codes(variant != "columns32")
    dm.stream_values(variant != "values8")
    x, r = x0.copy(), b.copy()
    it, _ = dm.solve(method, x, r, **(RR if method.endswith("rr") else {}))
    return dict(it=it, x=_bits(x), r=_bits(r), hist=_bits(B.last_history()),
                ctas=(dm.resident_ctas(), dm.coded_ctas(), dm.packed_ctas()))


def _same(got, want, what=""):
    assert got["it"] == want["it"], (what, got["it"], want["it"])
    assert got["ctas"] == want["ctas"], (what, got["ctas"], want["ctas"])
    assert got["hist"] == want["hist"], what
    assert got["x"] == want["x"] and got["r"] == want["r"], what


@pytest.mark.parametrize("src", ["numpy", "torch"])
@pytest.mark.parametrize("mega", [0, 1, 2])
@pytest.mark.parametrize("case", CASES)
def test_set_values_equals_fresh_handle(B, case, mega, src):
    """Solve, set new values, then every method with the default streams, 32-bit columns and 8-byte values, plus spmv and
    shift_residuals: all bit-identical to a handle created from the new values."""
    B.set_options(mega=mega, resident=1 if case == "resident" else 0)
    blk = _case_block(B, case)
    dv, ov = _values(blk)
    dv2, ov2 = _perturbed(dv, 2), _perturbed(ov, 2)
    n = blk.n_loc
    x0 = initial_guess("warm", n)
    dm = B.DeviceMatrix(blk)
    fresh = B.DeviceMatrix(_with_values(_case_block(B, case), dv2, ov2))
    try:
        b1 = dm.spmv(np.ones(n))
        _run(B, dm, "bicgstab", b1, x0)                           # a solve on the old values first
        dm.set_values(*_src(src, dv2, ov2))
        b = fresh.spmv(np.ones(n))
        assert _bits(dm.spmv(np.ones(n))) == _bits(b)
        for method in METHODS:
            for variant in VARIANTS:
                _same(_run(B, dm, method, b, x0, variant), _run(B, fresh, method, b, x0, variant), (case, mega, method, variant))
        sigma = np.array([0.0, 0.5, 1.5])
        xs = np.ascontiguousarray(np.tile(x0, (3, 1)))
        assert _bits(dm.shift_residuals(xs, b, sigma)) == _bits(fresh.shift_residuals(xs, b, sigma))
    finally:
        dm.destroy()
        fresh.destroy()


def test_value_tables_follow_the_values(B):
    """Rows of the first half scaled by 2^0 .. 2^19: their CTAs hold more than 16 sign / exponent fields and stream 8-byte
    values; back to the original values they pack again.  packed_ctas() and the results equal a fresh handle's at each step."""
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    dv, ov = _values(blk)
    row = np.repeat(np.arange(n), np.diff(blk.diag_arrays()[2].astype(np.int64)))
    dv2 = np.where(row < n // 2, dv * 2.0 ** (row % 20), dv)
    x0 = initial_guess("warm", n)
    dm = B.DeviceMatrix(blk)
    try:
        packed = []
        for step, vals in enumerate([dv, dv2, dv]):
            if step:
                dm.set_values(vals, None)
            fresh = B.DeviceMatrix(_with_values(_case_block(B, "stencil15"), vals, ov))
            try:
                b = fresh.spmv(np.ones(n))
                got, want = _run(B, dm, "bicgstab", b, x0), _run(B, fresh, "bicgstab", b, x0)
                _same(got, want, step)
                packed.append(got["ctas"][2])
            finally:
                fresh.destroy()
        assert packed[0] > 0 and 0 < packed[1] < packed[0] and packed[2] == packed[0], packed
    finally:
        dm.destroy()


def _shifted_sync(B, dm, method, x0s, b, sigma, seed, torch_vectors):
    torch = _torch()
    x, r = x0s.copy(), b.copy()
    if torch_vectors:
        x, r = torch.from_numpy(x).cuda(), torch.from_numpy(r).cuda()
    k, st = dm.shifted_solve(method, x, r, sigma, seed)
    seed_end, stop = B.last_shift_info(sigma.size)
    return dict(k=k, iters=st["iters"], seed=seed_end, stop=list(stop), x=_bits(x), r=_bits(r), hist=_bits(B.last_history()))


def _shifted_async(B, dm, method, x0s, b, sigma, seed):
    torch = _torch()
    x, r = torch.from_numpy(x0s.copy()).cuda(), torch.from_numpy(b.copy()).cuda()
    stop = torch.full((sigma.size,), -1, dtype=torch.int32, device="cuda")
    res = dm.shifted_solve_async(method, x, r, torch.from_numpy(sigma).cuda(), seed, stop_iter=stop)
    torch.cuda.synchronize()
    rec = B.decode_shift_result(res)
    return dict(k=rec["ret"], iters=rec["iters"], seed=rec["seed"], stop=list(stop.cpu().numpy()), x=_bits(x), r=_bits(r),
                hist=_bits(dm.shift_history()))


@pytest.mark.parametrize("method", SHIFTED)
def test_shifted_solvers_after_set_values(B, method):
    blk = _case_block(B, "resident")
    n = blk.n_loc
    dv, ov = _values(blk)
    dv2 = _perturbed(dv, 3)
    sigma, seed = np.array([0.0, 0.3, 1.1, 2.0]), 1
    x0s = initial_x_set(sigma.size, n)
    dm = B.DeviceMatrix(blk)
    fresh = B.DeviceMatrix(_with_values(_case_block(B, "resident"), dv2, ov))
    try:
        dm.shifted_solve(method, x0s.copy(), dm.spmv(np.ones(n)), sigma, seed)       # on the old values first
        dm.set_values(*_src("torch", dv2, ov))
        b = fresh.spmv(np.ones(n))
        for tv in (False, True):
            assert _shifted_sync(B, dm, method, x0s, b, sigma, seed, tv) == _shifted_sync(B, fresh, method, x0s, b, sigma, seed, tv)
        assert _shifted_async(B, dm, method, x0s, b, sigma, seed) == _shifted_async(B, fresh, method, x0s, b, sigma, seed)
    finally:
        dm.destroy()
        fresh.destroy()


def _fresh_async(B, blk, method, x0, b):
    """solve_async on a fresh handle of blk: x, r, record, history."""
    torch = _torch()
    dm = B.DeviceMatrix(blk)
    try:
        x, r = x0.clone(), b.clone()
        res = dm.solve_async(method, x, r)
        torch.cuda.synchronize()
        return dict(x=_bits(x), r=_bits(r), rec=B.decode_result(res), hist=_bits(dm.history()))
    finally:
        dm.destroy()


@pytest.mark.parametrize("mega", [0, 1])
def test_stream_order_without_host_synchronisation(B, mega):
    """solve_async (V1), set_values_async (V2), solve_async, all enqueued before any synchronisation, on one stream and with
    the update on a second stream; then the V2 buffer is overwritten after the update: nothing changes."""
    torch = _torch()
    B.set_options(mega=mega)
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    dv, ov = _values(blk)
    dv2 = _perturbed(dv, 4)
    x0 = torch.from_numpy(initial_guess("warm", n)).cuda()
    b = torch.ones(n, dtype=torch.float64, device="cuda")
    want1 = _fresh_async(B, _case_block(B, "stencil15"), "pipe_bicgstab", x0, b)
    want2 = _fresh_async(B, _with_values(_case_block(B, "stencil15"), dv2, ov), "pipe_bicgstab", x0, b)
    for second_stream in (False, True):
        dm = B.DeviceMatrix(blk)
        try:
            dm.prepare_async("pipe_bicgstab")
            s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
            buf = torch.from_numpy(dv2).cuda()
            x1, r1, x2, r2 = x0.clone(), b.clone(), x0.clone(), b.clone()
            torch.cuda.synchronize()
            res1 = dm.solve_async("pipe_bicgstab", x1, r1, stream=s)
            dm.set_values_async(buf, None, stream=s2 if second_stream else s)
            res2 = dm.solve_async("pipe_bicgstab", x2, r2, stream=s)
            torch.cuda.synchronize()
            got1 = dict(x=_bits(x1), r=_bits(r1), rec=B.decode_result(res1))
            got2 = dict(x=_bits(x2), r=_bits(r2), rec=B.decode_result(res2), hist=_bits(dm.history()))
            assert got1 == {k: want1[k] for k in got1}, second_stream
            assert got2 == want2, second_stream
            buf.fill_(-3.0)                                      # the stream has passed the update: the handle keeps V2
            x3, r3 = x0.clone(), b.clone()
            res3 = dm.solve_async("pipe_bicgstab", x3, r3, stream=s)
            torch.cuda.synchronize()
            assert dict(x=_bits(x3), r=_bits(r3), rec=B.decode_result(res3), hist=_bits(dm.history())) == want2
        finally:
            dm.destroy()


def test_captured_update_and_solve_replay(B):
    """One graph of {reset x, r; set_values_async(buf); solve_async} and one with shifted_solve_async, each replayed with buf
    holding V2, V3 and V4: every replay equals a fresh handle of those values."""
    torch = _torch()
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    dv, ov = _values(blk)
    sets = [_perturbed(dv, k) for k in (2, 3, 4)]
    x0 = torch.from_numpy(initial_guess("warm", n)).cuda()
    b = torch.ones(n, dtype=torch.float64, device="cuda")
    sigma = np.array([0.0, 0.4, 1.3])
    x0s = torch.from_numpy(initial_x_set(sigma.size, n)).cuda()
    sg = torch.from_numpy(sigma).cuda()
    method, smethod = "bicgstab", "shifted_lopbicgstab"
    dm = B.DeviceMatrix(blk)
    try:
        dm.prepare_async(method)
        dm.prepare_shifted_async(smethod, sigma.size)
        buf = torch.from_numpy(dv.copy()).cuda()
        x, r, res = x0.clone(), b.clone(), torch.zeros(24, dtype=torch.uint8, device="cuda")
        xs, rs = x0s.clone(), b.clone()
        sres = torch.zeros(32, dtype=torch.uint8, device="cuda")
        stop = torch.zeros(sigma.size, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        g, gs = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            x.copy_(x0)
            r.copy_(b)
            dm.set_values_async(buf)
            dm.solve_async(method, x, r, result=res)
        with torch.cuda.graph(gs):
            xs.copy_(x0s)
            rs.copy_(b)
            dm.set_values_async(buf)
            dm.shifted_solve_async(smethod, xs, rs, sg, 0, result=sres, stop_iter=stop)
        for vals in sets:
            buf.copy_(torch.from_numpy(vals))
            g.replay()
            torch.cuda.synchronize()
            got = dict(x=_bits(x), r=_bits(r), rec=B.decode_result(res), hist=_bits(dm.history()))
            fb = _with_values(_case_block(B, "stencil15"), vals, ov)
            assert got == _fresh_async(B, fb, method, x0, b)
            buf.copy_(torch.from_numpy(vals))
            gs.replay()
            torch.cuda.synchronize()
            got = dict(x=_bits(xs), r=_bits(rs), rec=B.decode_shift_result(sres), stop=list(stop.cpu().numpy()),
                       hist=_bits(dm.shift_history()))
            fresh = B.DeviceMatrix(fb)
            try:
                fx, fr = x0s.clone(), b.clone()
                fstop = torch.zeros(sigma.size, dtype=torch.int32, device="cuda")
                fres = fresh.shifted_solve_async(smethod, fx, fr, sg, 0, stop_iter=fstop)
                torch.cuda.synchronize()
                want = dict(x=_bits(fx), r=_bits(fr), rec=B.decode_shift_result(fres), stop=list(fstop.cpu().numpy()),
                            hist=_bits(fresh.shift_history()))
            finally:
                fresh.destroy()
            assert got == want
        del g, gs
    finally:
        dm.destroy()


@pytest.mark.parametrize("mega", [0, 1])
def test_shift_diagonal_equals_host_shift(B, mega):
    """shift_diagonal(0.75), then shift_diagonal(-0.125): each equals csr_shift_diagonal on the host blocks and a fresh handle."""
    B.set_options(mega=mega)
    blk = _case_block(B, "stencil15")
    n = blk.n_loc
    x0 = initial_guess("normal", n)
    b = np.ones(n)
    dm = B.DeviceMatrix(blk)
    ref = _case_block(B, "stencil15")
    try:
        for sigma in (0.75, -0.125):
            dm.shift_diagonal(sigma)
            B.lib.csr_shift_diagonal(C.byref(ref.diag), sigma)
            fresh = B.DeviceMatrix(ref)
            try:
                assert _bits(dm.spmv(x0)) == _bits(fresh.spmv(x0))
                for method in ("bicgstab", "pipe_bicgstab_rr"):
                    _same(_run(B, dm, method, b, x0), _run(B, fresh, method, b, x0), (sigma, method))
            finally:
                fresh.destroy()
    finally:
        dm.destroy()


def test_shift_diagonal_without_a_diagonal_entry_changes_nothing(B):
    n = 5000
    A = sp.diags([-np.ones(n - 1), 4.0 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], format="lil")
    A[77, 77] = 0.0
    A = sp.csr_matrix(A)
    A.eliminate_zeros()
    A.sort_indices()
    blk = B.blocks_from_csr(n, A.indptr, A.indices, A.data)
    x0 = initial_guess("warm", n)
    b = np.ones(n)
    dm = B.DeviceMatrix(blk)
    try:
        before = _run(B, dm, "bicgstab", b, x0)
        with pytest.raises(ValueError, match="no diagonal entry"):
            dm.shift_diagonal(1.0)
        with pytest.raises(ValueError, match="no diagonal entry"):
            dm.shift_diagonal(1.0)
        assert B.lib.bicg_matrix_shift_diagonal(dm.h, 1.0) == -1
        _same(_run(B, dm, "bicgstab", b, x0), before)
    finally:
        dm.destroy()
