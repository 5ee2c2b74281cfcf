"""GPU: shifted solves on the caller's CUDA stream (bicg_shifted_solve_async).  The asynchronous solve runs the kernels of
bicg_shifted_solve_dev in the same order, on the handle's workspace instead of per-call buffers, with its loop driven by a CUDA
WHILE node instead of the host.  So x_set, r, stop_iter, the result record and shift_history() must be bit-identical to the
synchronous solve of the same inputs on a fresh handle (its return value, bicg_stats, bicg_last_shift_info and
bicg_last_history), for all four methods: the shifted cases (a seed switch among them), L = 1 and L on both sides of the
shared-memory pass edges of sh_vec_shift (945 / 946) and lop_vec_update (969 / 970), converged and cut at SHIFT_MAX_ITER = 3
(not a multiple of the 8 iterations per loop body), odd n_loc with x_set at a one-element offset.  The call must not wait for
the stream, calls on one handle must be ordered against every other entry point, and a captured solve must replay with new b and
sigma, also after its workspace was outgrown."""
import ctypes as C

import numpy as np
import pytest

from helpers import global_csr, initial_x_set
from shifted_fixed_cases import FIXED_CASES
from shifted_lop_cases import SHIFTED_LOP_CASES, shifted_lop_problem

pytestmark = pytest.mark.gpu
METHODS = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]
CASES = SHIFTED_LOP_CASES + [c[:7] for c in FIXED_CASES[len(SHIFTED_LOP_CASES):]]
STOPS = {"converged": 1000, "cut3": 3}
EDGES = [1, 945, 946, 969, 970]


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, shift_tol=1e-12, shift_max_iter=1000, shift_error=0)
    yield
    B.set_options(shift_tol=1e-12, shift_max_iter=1000)


def _torch():
    import torch
    return torch


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def _sync(B, blk, method, x0, b, sigma, seed):
    """bicg_shifted_solve_dev on a fresh handle: x_set, r, the record the asynchronous solve must write, stop_iter, history."""
    torch = _torch()
    dm = B.DeviceMatrix(blk)
    try:
        x, r = torch.from_numpy(x0.copy()).cuda(), torch.from_numpy(b.copy()).cuda()
        k, st = dm.shifted_solve(method, x, r, sigma, seed)
        seed_end, stop = B.last_shift_info(sigma.size)
        rec = {"ret": k, "iters": st["iters"], "converged": st["converged"], "seed": seed_end, "error": 0, "final_res": st["final_res"]}
        return dict(x=_bits(x), r=_bits(r), rec=rec, stop=np.asarray(stop, dtype=np.int32), hist=_bits(B.last_history()))
    finally:
        dm.destroy()


def _got(B, dm, x, r, res, stop):
    return dict(x=_bits(x), r=_bits(r), rec=B.decode_shift_result(res), stop=stop.cpu().numpy(), hist=_bits(dm.shift_history()))


def _same(got, want, what=""):
    gr, wr = got["rec"], want["rec"]
    for key in ("ret", "iters", "converged", "seed", "error"):
        assert gr[key] == wr[key], (what, key, gr, wr)
    assert _bits(gr["final_res"]) == _bits(wr["final_res"]), (what, gr, wr)
    assert np.array_equal(got["stop"], want["stop"]), what
    assert got["hist"] == want["hist"], what
    assert got["x"] == want["x"] and got["r"] == want["r"], what


def _async(B, dm, method, x0, b, sigma, seed, offset=False, stream=None):
    """One asynchronous solve on CUDA tensors (x_set at a one-element offset when asked), then a device synchronise."""
    torch = _torch()
    L, n = x0.shape
    if offset:
        big = torch.full((L * n + 2,), 7.0, dtype=torch.float64, device="cuda")
        x = big[1:1 + L * n].view(L, n)
        x.copy_(torch.from_numpy(x0))
    else:
        big, x = None, torch.from_numpy(x0.copy()).cuda()
    r = torch.from_numpy(b.copy()).cuda()
    sg = torch.from_numpy(sigma).cuda()
    stop = torch.full((L,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    res = dm.shifted_solve_async(method, x, r, sg, seed, stop_iter=stop, stream=stream)
    torch.cuda.synchronize()
    if big is not None:
        assert big[0].item() == 7.0 and big[-1].item() == 7.0                 # nothing written outside x_set
    return _got(B, dm, x, r, res, stop)


def _case_problem(B, O, case):
    blk, n, ptr, col, val = global_csr(B, *case[1:4])
    sigma, b, seed = shifted_lop_problem(O, n, ptr, col, val, case)
    return blk, n, sigma, b, seed


@pytest.mark.parametrize("stop", list(STOPS))
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_async_bit_identical_to_sync(B, O, case, method, stop):
    B.set_options(shift_max_iter=STOPS[stop])
    blk, n, sigma, b, seed = _case_problem(B, O, case)
    x0 = initial_x_set(sigma.size, n)
    want = _sync(B, blk, method, x0, b, sigma, seed)
    dm = B.DeviceMatrix(blk)
    try:
        got = _async(B, dm, method, x0, b, sigma, seed)
    finally:
        dm.destroy()
    _same(got, want, (case[0], method, stop))
    if stop == "cut3":
        assert want["rec"]["iters"] <= 3
    if case[0] == "sh_convdiff_g40_L6_switch" and method == "shifted_lopbicg_switching" and stop == "converged":
        assert got["rec"]["seed"] != seed                                       # the seed does switch


@pytest.mark.parametrize("L", EDGES)
@pytest.mark.parametrize("method", METHODS)
def test_async_pass_edges_odd_n_offset(B, O, method, L):
    """random n = 3001 (odd: every other block of the view is misaligned), x_set at a one-element offset, nonzero x0."""
    blk, n, ptr, col, val = global_csr(B, "random", 3001, 8)
    seed = L // 2
    sigma = (np.arange(L) + 1) * (0.05 / L)
    b = O.spmv(n, ptr, col, val, np.ones(n)); O.daxpy(sigma[seed], np.ones(n), b)
    x0 = initial_x_set(L, n)
    want = _sync(B, blk, method, x0, b, sigma, seed)
    dm = B.DeviceMatrix(blk)
    try:
        got = _async(B, dm, method, x0, b, sigma, seed, offset=True)
    finally:
        dm.destroy()
    _same(got, want, (method, L))


def test_async_does_not_wait_for_the_stream(B, O):
    """A second of device sleep on a side stream, then b written behind it, then the call: it returns while the stream is still
    busy, and the solve reads the b written behind the sleep."""
    torch = _torch()
    blk, n, sigma, b, seed = _case_problem(B, O, SHIFTED_LOP_CASES[1])
    x0 = initial_x_set(sigma.size, n)
    want = _sync(B, blk, "shifted_lopbicg_switching", x0, b, sigma, seed)
    dm = B.DeviceMatrix(blk)
    try:
        dm.prepare_shifted_async("shifted_lopbicg_switching", sigma.size)
        s = torch.cuda.Stream()
        x, r = torch.from_numpy(x0.copy()).cuda(), torch.zeros(n, dtype=torch.float64, device="cuda")
        bt, sg = torch.from_numpy(b).cuda(), torch.from_numpy(sigma).cuda()
        stop = torch.zeros(sigma.size, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(int(2e9))                            # ~1 s at the H100's clock
            r.copy_(bt)
            res = dm.shifted_solve_async("shifted_lopbicg_switching", x, r, sg, seed, stop_iter=stop)
        assert not s.query()
        s.synchronize()
        got = _got(B, dm, x, r, res, stop)
    finally:
        dm.destroy()
    _same(got, want)


def test_async_calls_on_one_handle_are_ordered(B, O):
    """Two streams on one handle with no host synchronisation between them; then an asynchronous shifted solve followed at once by
    a synchronous plain solve, an asynchronous plain solve and a synchronous shifted solve, all on the same handle (they share its
    arena vectors).  Every result equals its sequential counterpart."""
    torch = _torch()
    case = SHIFTED_LOP_CASES[0]
    blk, n, sigma, b, seed = _case_problem(B, O, case)
    b2 = b * 0.5 + 1.0
    x0 = initial_x_set(sigma.size, n)
    m1, m2 = "shifted_lopbicgstab", "shifted_lopbicg"
    want1, want2 = _sync(B, blk, m1, x0, b, sigma, seed), _sync(B, blk, m2, x0, b2, sigma, seed)
    bt = torch.from_numpy(b).cuda()
    B.set_options(tol=1e-10, max_iter=1000)
    ref = B.DeviceMatrix(blk)
    try:
        xp, rp = torch.zeros_like(bt), bt.clone()
        it_p, st_p = ref.solve("bicgstab", xp, rp)
        want_plain = (_bits(xp), _bits(rp), _bits(B.last_history()), it_p, _bits(st_p["final_res"]))
    finally:
        ref.destroy()
    dm = B.DeviceMatrix(blk)
    try:
        sg = torch.from_numpy(sigma).cuda()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        x1, r1 = torch.from_numpy(x0.copy()).cuda(), bt.clone()
        x2, r2 = torch.from_numpy(x0.copy()).cuda(), torch.from_numpy(b2).cuda()
        st1, st2 = (torch.zeros(sigma.size, dtype=torch.int32, device="cuda") for _ in range(2))
        dm.prepare_shifted_async(m1, sigma.size); dm.prepare_shifted_async(m2, sigma.size)
        torch.cuda.synchronize()
        res1 = dm.shifted_solve_async(m1, x1, r1, sg, seed, stop_iter=st1, stream=s1)
        res2 = dm.shifted_solve_async(m2, x2, r2, sg, seed, stop_iter=st2, stream=s2)
        s2.synchronize()
        _same(_got(B, dm, x2, r2, res2, st2), want2, "second of two streams")
        s1.synchronize()
        got1 = _got(B, dm, x1, r1, res1, st1)
        got1["hist"] = want1["hist"]                               # the handle's history is the second solve's now
        _same(got1, want1, "first of two streams")

        # asynchronous shifted, synchronous plain, asynchronous plain, synchronous shifted: no synchronise in between
        x3, r3 = torch.from_numpy(x0.copy()).cuda(), bt.clone()
        st3 = torch.zeros(sigma.size, dtype=torch.int32, device="cuda")
        xp, rp = torch.zeros_like(bt), bt.clone()
        xa, ra = torch.zeros_like(bt), bt.clone()
        x4, r4 = torch.from_numpy(x0.copy()).cuda(), torch.from_numpy(b2).cuda()
        torch.cuda.synchronize()
        res3 = dm.shifted_solve_async(m1, x3, r3, sg, seed, stop_iter=st3)
        it_p, st_p = dm.solve("bicgstab", xp, rp)                 # waits for the shifted solve on this handle
        got_plain = (_bits(xp), _bits(rp), _bits(B.last_history()), it_p, _bits(st_p["final_res"]))
        resa = dm.solve_async("bicgstab", xa, ra)
        k4, stats4 = dm.shifted_solve(m2, x4, r4, sigma, seed)
        hist4 = _bits(B.last_history())
        torch.cuda.synchronize()
        got3 = _got(B, dm, x3, r3, res3, st3)
        got3["hist"] = want1["hist"]
        _same(got3, want1, "asynchronous shifted first")
        assert got_plain == want_plain, "synchronous plain after asynchronous shifted"
        rec = B.decode_result(resa)
        assert (_bits(xa), _bits(ra), rec["iters"], _bits(rec["final_res"])) == \
            (want_plain[0], want_plain[1], want_plain[3], want_plain[4]), "asynchronous plain"
        assert k4 == want2["rec"]["ret"] and _bits(x4) == want2["x"] and _bits(r4) == want2["r"] and hist4 == want2["hist"], \
            "synchronous shifted last"
        assert _bits(stats4["final_res"]) == _bits(want2["rec"]["final_res"])
    finally:
        dm.destroy()
        B.set_options(tol=1e-15, max_iter=1000)


def _capture(B, dm, method, L, n, seed):
    """{r <- b_buf; x_set <- x0_buf; shifted_solve_async} captured into a torch CUDA graph; returns the graph and its buffers."""
    torch = _torch()
    f64 = dict(dtype=torch.float64, device="cuda")
    bufs = dict(b=torch.zeros(n, **f64), x0=torch.zeros(L, n, **f64), x=torch.zeros(L, n, **f64), r=torch.zeros(n, **f64),
                sigma=torch.zeros(L, **f64), stop=torch.zeros(L, dtype=torch.int32, device="cuda"),
                res=torch.zeros(32, dtype=torch.uint8, device="cuda"))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        bufs["r"].copy_(bufs["b"])
        bufs["x"].copy_(bufs["x0"])
        dm.shifted_solve_async(method, bufs["x"], bufs["r"], bufs["sigma"], seed, result=bufs["res"], stop_iter=bufs["stop"])
    return g, bufs


def _replay(B, dm, g, bufs, x0, b, sigma):
    torch = _torch()
    bufs["b"].copy_(torch.from_numpy(b)); bufs["x0"].copy_(torch.from_numpy(x0)); bufs["sigma"].copy_(torch.from_numpy(sigma))
    g.replay()
    torch.cuda.synchronize()
    return _got(B, dm, bufs["x"], bufs["r"], bufs["res"], bufs["stop"])


@pytest.mark.parametrize("method", METHODS)
def test_captured_solve_replays(B, O, method):
    """Three replays with different b and sigma, each equal to a fresh synchronous solve of those inputs."""
    case = SHIFTED_LOP_CASES[1]                                    # convdiff g40, 6 shifts: the switching solver switches
    blk, n, sigma, b, seed = _case_problem(B, O, case)
    x0 = initial_x_set(sigma.size, n)
    inputs = [(b, sigma), (b * 0.5 + 1.0, sigma * 0.75), (b - 0.25, sigma + 0.05)]
    wants = [_sync(B, blk, method, x0, bb, sg, seed) for bb, sg in inputs]
    dm = B.DeviceMatrix(blk)
    try:
        dm.prepare_shifted_async(method, sigma.size)
        g, bufs = _capture(B, dm, method, sigma.size, n, seed)
        for i, (bb, sg) in enumerate(inputs):
            _same(_replay(B, dm, g, bufs, x0, bb, sg), wants[i], (method, i))
        del g
    finally:
        dm.destroy()


def test_capture_returns_minus_2_when_unprepared(B, O):
    """Without prepare, and prepared for another sigma_len: -2, and the capture stays usable."""
    torch = _torch()
    blk, n, sigma, b, seed = _case_problem(B, O, SHIFTED_LOP_CASES[0])
    L = sigma.size
    dm = B.DeviceMatrix(blk)
    try:
        f64 = dict(dtype=torch.float64, device="cuda")
        x, r, sg = torch.zeros(L, n, **f64), torch.from_numpy(b).cuda(), torch.from_numpy(sigma).cuda()
        res = torch.zeros(32, dtype=torch.uint8, device="cuda")
        args = lambda m, LL: (dm.h, B.SHIFTED_SOLVE_EX[m], C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()),
                              C.c_void_p(sg.data_ptr()), LL, 0, C.c_void_p(torch.cuda.current_stream().cuda_stream),
                              C.c_void_p(res.data_ptr()), None)
        for prepared in (None, L + 1):
            if prepared:
                dm.prepare_shifted_async("shifted_lopbicgstab", prepared)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                r.mul_(2.0)
                rc = B.lib.bicg_shifted_solve_async(*args("shifted_lopbicgstab", L))
            assert rc == -2, (prepared, rc)
            g.replay()
            torch.cuda.synchronize()
            assert bool((r == torch.from_numpy(b).cuda() * 2.0).all())
            r.copy_(torch.from_numpy(b))
            del g
        with pytest.raises(RuntimeError):
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2):
                dm.shifted_solve_async("shifted_pipe_lopbicgstab", x, r, sg, seed, result=res)
        # null pointers, unknown methods, bad sigma_len / seed are refused before anything is enqueued
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        xp, rp, sp_ = C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()), C.c_void_p(sg.data_ptr())
        for bad in [(None, rp, sp_, L, 0, 1), (xp, None, sp_, L, 0, 1), (xp, rp, None, L, 0, 1), (xp, rp, sp_, 0, 0, 1),
                    (xp, rp, sp_, L, L, 1), (xp, rp, sp_, L, -1, 1), (xp, rp, sp_, L, 0, 7)]:
            bx, br, bs, bl, bseed, bm = bad
            assert B.lib.bicg_shifted_solve_async(dm.h, bm, bx, br, bs, bl, bseed, s, None, None) == -1, bad
        assert B.lib.bicg_shifted_solve_async_prepare(dm.h, 7, L) == -1
        assert B.lib.bicg_shifted_solve_async_prepare(dm.h, 1, 0) == -1
    finally:
        dm.destroy()


@pytest.mark.parametrize("captured", [False, True])
def test_first_call_on_a_fresh_handle(B, O, captured):
    """bicg_matrix_create returns with work in flight on the library's stream; here a second of device sleep and the write of b
    follow it there.  The first asynchronous shifted call on the handle, captured or not, runs behind both."""
    torch = _torch()
    method = "shifted_pipe_lopbicgstab"
    blk, n, sigma, b, seed = _case_problem(B, O, SHIFTED_LOP_CASES[0])
    L = sigma.size
    x0 = initial_x_set(L, n)
    want = _sync(B, blk, method, x0, b, sigma, seed)
    dm = B.DeviceMatrix(blk)
    try:
        x, r = torch.from_numpy(x0.copy()).cuda(), torch.zeros(n, dtype=torch.float64, device="cuda")
        bt, sg = torch.from_numpy(b).cuda(), torch.from_numpy(sigma).cuda()
        stop = torch.zeros(L, dtype=torch.int32, device="cuda")
        res = torch.zeros(32, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        lib_stream = torch.cuda.ExternalStream(B.lib.bicg_stream())
        with torch.cuda.stream(lib_stream):
            torch.cuda._sleep(int(2e9))
            r.copy_(bt)
        s = torch.cuda.Stream()
        if captured:
            dm.prepare_shifted_async(method, L)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                g.capture_begin()
                dm.shifted_solve_async(method, x, r, sg, seed, result=res, stop_iter=stop)
                g.capture_end()
                g.replay()
        else:
            dm.shifted_solve_async(method, x, r, sg, seed, result=res, stop_iter=stop, stream=s)
        assert not s.query()
        s.synchronize()
        got = _got(B, dm, x, r, res, stop)
    finally:
        dm.destroy()
    _same(got, want, captured)


def test_outgrown_workspace_keeps_the_old_graph_working(B, O):
    """Capture at SHIFT_MAX_ITER = 5, then raise it to 1000 and re-prepare: the workspace is replaced, the earlier graph still
    replays correctly on the retired one (its captured SHIFT_MAX_ITER), and a new capture uses the new workspace."""
    method = "shifted_lopbicg_switching"
    blk, n, sigma, b, seed = _case_problem(B, O, SHIFTED_LOP_CASES[1])
    L = sigma.size
    x0 = initial_x_set(L, n)
    B.set_options(shift_max_iter=5)
    want_cut = _sync(B, blk, method, x0, b, sigma, seed)
    B.set_options(shift_max_iter=1000)
    want_full = _sync(B, blk, method, x0, b * 0.5 + 1.0, sigma, seed)
    dm = B.DeviceMatrix(blk)
    try:
        B.set_options(shift_max_iter=5)
        dm.prepare_shifted_async(method, L)
        g_old, bufs_old = _capture(B, dm, method, L, n, seed)
        B.set_options(shift_max_iter=1000)
        dm.prepare_shifted_async(method, L)
        g_new, bufs_new = _capture(B, dm, method, L, n, seed)
        _same(_replay(B, dm, g_old, bufs_old, x0, b, sigma), want_cut, "old graph")
        _same(_replay(B, dm, g_new, bufs_new, x0, b * 0.5 + 1.0, sigma), want_full, "new graph")
        _same(_replay(B, dm, g_old, bufs_old, x0, b, sigma), want_cut, "old graph again")
        del g_old, g_new
    finally:
        dm.destroy()
