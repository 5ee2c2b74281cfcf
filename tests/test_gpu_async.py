"""GPU: solves on the caller's CUDA stream (bicg_solve_async).  An asynchronous solve runs the same kernels in the same order as
bicg_solve, so x, r, the history (bicg_matrix_history) and the bicg_result record must be bit-identical to the synchronous solve
with device vectors, on every loop path: the persistent kernel (resident; streaming with 16-bit codes and packed values) and the
kernel-per-phase path whose loop a CUDA WHILE node drives on the device (BICG_MEGA=0, and the default for long rows).  The call
must not wait for the stream, two calls on one handle must be ordered, and a solve captured into a CUDA graph must give the
synchronous result for the b of every replay."""
import ctypes as C

import numpy as np
import pytest

from helpers import METHODS, initial_guess

pytestmark = pytest.mark.gpu

RR = dict(krr=10, nrr=3)
# path -> options; "graph" runs the kernel-per-phase kernels, "resident" / "streaming" the persistent kernel
PATHS = {"resident": dict(mega=1, resident=1), "streaming": dict(mega=1, resident=0), "graph": dict(mega=0, resident=1)}
# stop -> (tol, max_iter): converged, or cut at max_iter (37 is not a multiple of the 10 iterations per graph batch; PIPE_RR's
# replacements at 10, 20, 30 lie inside krr * nrr = 30, and iterations 31..36 past it)
STOPS = {"converged": (1e-10, 1000), "max_iter": (0.0, 37)}


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, mega=1, resident=1, tol=1e-10, max_iter=1000)
    yield
    B.set_options(mega=1, resident=1, tol=1e-15, max_iter=1000)


def _torch():
    import torch
    return torch


def _problem(B, kind, g, p0, x0_kind):
    torch = _torch()
    blk = B.gen_block(kind, g, p0)
    n = blk.n_loc
    b = torch.from_numpy(_spmv_ones(B, blk)).cuda()
    x0 = torch.zeros(n, dtype=torch.float64, device="cuda") if x0_kind == "zero" else \
        torch.from_numpy(initial_guess(x0_kind, n)).cuda()
    return blk, x0, b


def _spmv_ones(B, blk):
    dm = B.DeviceMatrix(blk)
    try:
        return dm.spmv(np.ones(blk.n_loc))
    finally:
        dm.destroy()


def _sync(B, dm, method, x0, b):
    """bicg_solve with device vectors: (x, r, history, record) -- the record as the bicg_result fields of its stats."""
    x, r = x0.clone(), b.clone()
    kw = RR if method.endswith("rr") else {}
    it, st = dm.solve(method, x, r, **kw)
    hist = B.last_history()
    assert np.array_equal(dm.history(), hist)
    return x, r, hist, {"iters": it, "converged": st["converged"], "error": 0, "final_res": st["final_res"]}


def _async(B, dm, method, x0, b, stream=None):
    torch = _torch()
    x, r = x0.clone(), b.clone()
    kw = RR if method.endswith("rr") else {}
    res = dm.solve_async(method, x, r, stream=stream, **kw)
    torch.cuda.synchronize()
    return x, r, dm.history(), B.decode_result(res)


def _same(got, want, what=""):
    gx, gr, gh, grec = got
    wx, wr, wh, wrec = want
    assert np.array_equal(gh, wh), (what, gh[:5], wh[:5], len(gh), len(wh))
    assert grec["iters"] == wrec["iters"] and grec["converged"] == wrec["converged"] and grec["error"] == 0, (what, grec, wrec)
    assert np.float64(grec["final_res"]).tobytes() == np.float64(wrec["final_res"]).tobytes(), (what, grec, wrec)
    assert bool((gx == wx).all()) and bool((gr == wr).all()), what


@pytest.mark.parametrize("stop", list(STOPS))
@pytest.mark.parametrize("x0_kind", ["zero", "normal"])
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("path", list(PATHS))
def test_async_bit_identical_to_sync(B, path, method, x0_kind, stop):
    tol, max_iter = STOPS[stop]
    B.set_options(tol=tol, max_iter=max_iter, **PATHS[path])
    blk, x0, b = _problem(B, "stencil15", 12, 14.0, x0_kind)
    ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
    try:
        want = _sync(B, ref_dm, method, x0, b)
        got = _async(B, dm, method, x0, b)
        if path != "graph":
            assert dm.resident_ctas() == ref_dm.resident_ctas() and (dm.resident_ctas() > 0) == (path == "resident")
            assert dm.packed_ctas() == ref_dm.packed_ctas() and (dm.packed_ctas() > 0) == (path == "streaming")
    finally:
        ref_dm.destroy(); dm.destroy()
    _same(got, want, (path, method, x0_kind, stop))
    assert (want[3]["converged"] == 1) == (stop == "converged")
    if stop == "max_iter":
        assert want[3]["iters"] == max_iter


@pytest.mark.parametrize("method", METHODS)
def test_async_random_long_rows_kernel_per_phase(B, method):
    """random, k = 32 at 1 M rows: the default plan runs the kernel-per-phase path (long rows), from x0 != 0, cut at max_iter."""
    B.set_options(tol=0.0, max_iter=25)
    blk, x0, b = _problem(B, "random", 1 << 20, 32, "warm")
    ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
    try:
        want = _sync(B, ref_dm, method, x0, b)
        assert B.last_stats()["kernel_launches"] > 20            # the loop ran one kernel per phase
        got = _async(B, dm, method, x0, b)
    finally:
        ref_dm.destroy(); dm.destroy()
    _same(got, want, method)


@pytest.mark.parametrize("path", ["resident", "graph"])
def test_async_does_not_wait_for_the_stream(B, path):
    """A second of device sleep on a side stream, then b written behind it, then the solve: the call returns while the stream is
    still busy, and the solve reads the b written behind the sleep."""
    torch = _torch()
    B.set_options(**PATHS[path])
    blk, x0, b = _problem(B, "stencil15", 12, 14.0, "zero")
    ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
    try:
        want = _sync(B, ref_dm, "bicgstab", x0, b)
        dm.prepare_async("bicgstab")
        s = torch.cuda.Stream()
        x = torch.zeros_like(b)
        r = torch.zeros_like(b)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(int(2e9))                            # ~1 s at the H100's clock
            r.copy_(b)
            res = dm.solve_async("bicgstab", x, r)
        assert not s.query()
        s.synchronize()
        got = (x, r, dm.history(), B.decode_result(res))
    finally:
        ref_dm.destroy(); dm.destroy()
    _same(got, want, path)


@pytest.mark.parametrize("path", ["resident", "graph"])
def test_async_calls_on_one_handle_are_ordered(B, path):
    """Two streams, one handle, two b, no host synchronisation between the calls; then an asynchronous call followed at once by
    a synchronous one on the same handle.  Every result equals the sequential synchronous one."""
    torch = _torch()
    B.set_options(**PATHS[path])
    blk, x0, b1 = _problem(B, "stencil15", 12, 14.0, "zero")
    b2 = b1 * 0.5 + 1.0
    b3 = b1 - 0.25
    ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
    try:
        want = [_sync(B, ref_dm, "pipe_bicgstab", x0, bb) for bb in (b1, b2, b3)]
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        x1, r1, x2, r2 = x0.clone(), b1.clone(), x0.clone(), b2.clone()
        torch.cuda.synchronize()
        res1 = dm.solve_async("pipe_bicgstab", x1, r1, stream=s1)
        res2 = dm.solve_async("pipe_bicgstab", x2, r2, stream=s2)
        s2.synchronize()
        got2 = (x2, r2, dm.history(), B.decode_result(res2))
        s1.synchronize()
        got1 = (x1, r1, None, B.decode_result(res1))
        _same((got1[0], got1[1], want[0][2], got1[3]), want[0], "first of two streams")
        _same(got2, want[1], "second of two streams")

        x3, r3 = x0.clone(), b3.clone()
        torch.cuda.synchronize()
        res3 = dm.solve_async("pipe_bicgstab", x3, r3)
        got_sync = _sync(B, dm, "pipe_bicgstab", x0, b1)          # waits for the asynchronous solve on this handle
        torch.cuda.synchronize()
        _same((x3, r3, want[2][2], B.decode_result(res3)), want[2], "asynchronous before synchronous")
        _same(got_sync, want[0], "synchronous after asynchronous")
    finally:
        ref_dm.destroy(); dm.destroy()


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("path", ["resident", "graph"])
def test_captured_solve_replays(B, path, method):
    """{r <- b_buf; x <- 0; solve_async} captured into a torch CUDA graph, replayed with three different b."""
    torch = _torch()
    B.set_options(**PATHS[path])
    blk, x0, b = _problem(B, "stencil15", 12, 14.0, "zero")
    bs = [b, b * 0.5 + 1.0, b - 0.25]
    kw = RR if method.endswith("rr") else {}
    ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
    try:
        want = [_sync(B, ref_dm, method, x0, bb) for bb in bs]
        dm.prepare_async(method)
        b_buf, x, r = torch.zeros_like(b), torch.zeros_like(b), torch.zeros_like(b)
        res = torch.zeros(24, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            r.copy_(b_buf)
            x.zero_()
            dm.solve_async(method, x, r, result=res, **kw)
        for i, bb in enumerate(bs):
            b_buf.copy_(bb)
            g.replay()
            torch.cuda.synchronize()
            _same((x, r, dm.history(), B.decode_result(res)), want[i], (path, method, i))
        del g
    finally:
        ref_dm.destroy(); dm.destroy()


def test_capture_without_prepare_returns_minus_2(B):
    torch = _torch()
    blk, x0, b = _problem(B, "stencil15", 12, 14.0, "zero")
    dm = B.DeviceMatrix(blk)
    try:
        x, r = x0.clone(), b.clone()
        res = torch.zeros(24, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            r.mul_(1.0)
            rc = B.lib.bicg_solve_async(dm.h, 0, C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), 0, 0,
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_void_p(res.data_ptr()))
        assert rc == -2
        g.replay()
        torch.cuda.synchronize()
        assert bool((r == b).all())
        with pytest.raises(RuntimeError):
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2):
                dm.solve_async("ca_bicgstab", x, r, result=res)
        # null vectors and unknown methods are refused before anything is enqueued
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert B.lib.bicg_solve_async(dm.h, 0, None, C.c_void_p(r.data_ptr()), 0, 0, s, None) == -1
        assert B.lib.bicg_solve_async(dm.h, 7, C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), 0, 0, s, None) == -1
    finally:
        dm.destroy()


@pytest.mark.parametrize("captured", [False, True])
@pytest.mark.parametrize("path", ["resident", "graph"])
def test_first_call_on_a_fresh_handle_waits_for_the_library_stream(B, path, captured):
    """bicg_matrix_create returns with work still in flight on the library's stream.  The first asynchronous call on a handle,
    captured or not, must run behind it.  Here that work is a second of device sleep followed by the write of b into r, enqueued
    on the library's stream (bicg_stream) after the handle was created; nothing synchronises before the call."""
    torch = _torch()
    B.set_options(**PATHS[path])
    blk, x0, b = _problem(B, "stencil15", 12, 14.0, "zero")
    ref_dm = B.DeviceMatrix(blk)
    try:
        want = _sync(B, ref_dm, "bicgstab", x0, b)
    finally:
        ref_dm.destroy()
    dm = B.DeviceMatrix(blk)
    try:
        x, r = torch.zeros_like(b), torch.zeros_like(b)
        res = torch.zeros(24, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        lib_stream = torch.cuda.ExternalStream(B.lib.bicg_stream())
        with torch.cuda.stream(lib_stream):
            torch.cuda._sleep(int(2e9))                            # ~1 s at the H100's clock
            r.copy_(b)
        s = torch.cuda.Stream()
        if captured:
            dm.prepare_async("bicgstab")
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                g.capture_begin()
                dm.solve_async("bicgstab", x, r, result=res)
                g.capture_end()
                g.replay()
        else:
            dm.solve_async("bicgstab", x, r, result=res, stream=s)
        assert not s.query()                                       # queued behind the sleep, not run before it
        s.synchronize()
        got = (x, r, dm.history(), B.decode_result(res))
    finally:
        dm.destroy()
    _same(got, want, (path, captured))


@pytest.mark.parametrize("captured", [False, True])
def test_first_call_on_a_freshly_uploaded_transport_handle(B, captured):
    """T' at g = 117 (1.6 M rows): a second handle of a shape already tuned uploads and encodes the matrix on the library's
    stream without waiting for it; solve_async (or prepare, capture, replay) follows at once on another stream."""
    torch = _torch()
    B.set_options(tol=0.0, max_iter=30)
    blk, x0, b = _problem(B, "stencil15", 117, 14.0, "zero")
    ref_dm = B.DeviceMatrix(blk)
    try:
        want = _sync(B, ref_dm, "bicgstab", x0, b)
    finally:
        ref_dm.destroy()
    x, r = torch.zeros_like(b), b.clone()
    res = torch.zeros(24, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    dm = B.DeviceMatrix(blk)
    try:
        if captured:
            dm.prepare_async("bicgstab")
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                g.capture_begin()
                dm.solve_async("bicgstab", x, r, result=res)
                g.capture_end()
                g.replay()
        else:
            dm.solve_async("bicgstab", x, r, result=res, stream=s)
        s.synchronize()
        got = (x, r, dm.history(), B.decode_result(res))
    finally:
        dm.destroy()
    _same(got, want, captured)


def test_decode_result_waits_for_the_given_stream(B):
    torch = _torch()
    blk, x0, b = _problem(B, "stencil15", 12, 14.0, "zero")
    ref_dm, dm = B.DeviceMatrix(blk), B.DeviceMatrix(blk)
    try:
        want = _sync(B, ref_dm, "bicgstab", x0, b)
        s = torch.cuda.Stream()
        x, r = x0.clone(), b.clone()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(int(1e9))
        res = dm.solve_async("bicgstab", x, r, stream=s)
        rec = B.decode_result(res, stream=s)
    finally:
        ref_dm.destroy(); dm.destroy()
    assert rec["iters"] == want[3]["iters"] and rec["converged"] == 1, rec
