"""GPU: loss.backward() through shifted solves (shifted_solve_autograd) and shifts of products (multiply_autograd's sigma), and
the two device operations their backward adds: the diagonal shift by a device-resident sigma (shift_diagonal_async) and batched
global dot products in a pinned order (dots_async).  For X_j = (A + sigma_j I)^-1 b the backward solves (A^T + sigma_j I)
lambda_j = dL/dX_j on the refreshed and shifted transpose, one shift after another.
Checked: against dense numpy, with torch.autograd.gradcheck, bit for bit against the explicit sequence refresh -> shift -> solve
and against fresh handles of host-shifted transposed blocks on every shifted method and loop path; the shift against host
shifts; the dots bit for bit against a CPU model of their order; zero and partial losses, stale handles, interleaved forwards,
side streams, CUDA graph replays, convergence records and argument errors."""
import ctypes as C

import numpy as np
import pytest

from rowsum_model import fma
from test_gpu_autograd import _bits, _cuda, _perturbed, small_csr
from test_gpu_transpose import _case_csr, _same_everywhere, transposed_csr

pytestmark = pytest.mark.gpu

SIGMA = np.array([0.0, 0.5, 1.25, -0.125])


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, tol=1e-10, max_iter=1000, shift_tol=1e-12, shift_max_iter=1000, mega=1, resident=1)
    yield
    B.set_options(tol=1e-15, max_iter=1000, shift_tol=1e-12, shift_max_iter=1000, mega=1, resident=1)


def _torch():
    import torch
    return torch


def _handle(B, n, ptr, col, val):
    return B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))


def _host_shifted(B, n, ptr, col, val, sigmas):
    """a fresh handle of the blocks of (ptr, col, val) after csr_shift_diagonal by every sigma in turn"""
    blk = B.blocks_from_csr(n, ptr, col, val)
    for s in sigmas:
        B.lib.csr_shift_diagonal(C.byref(blk.diag), float(s))
    return B.DeviceMatrix(blk)


def _has_diagonal(n, ptr, col):
    rows = np.repeat(np.arange(n), np.diff(ptr))
    return np.unique(rows[col == rows]).size == n


def _shifted_grads(B, dm, method, b, sigma, vals, w, **kw):
    """X, b.grad, sigma.grad and vals.grad of loss = (w * X).sum() with X = shifted_solve_autograd(dm, b, sigma, ...)"""
    tb, ts, tv = _cuda(b, True), _cuda(sigma, True), _cuda(vals, True)
    x = B.shifted_solve_autograd(dm, tb, ts, method, diag_val=tv, **kw)
    (x * _cuda(w)).sum().backward()
    return x.detach(), tb.grad, ts.grad, tv.grad


def _dense(n, ptr, col, vals):
    A = np.zeros((n, n))
    np.add.at(A, (np.repeat(np.arange(n), np.diff(ptr)), col), vals)
    return A


@pytest.mark.parametrize("method", ["shifted_lopbicg_switching", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab",
                                    "shifted_lopbicg"])
@pytest.mark.parametrize("case", ["convdiff", "golden", "tprime8"])
def test_against_dense_numpy(B, case, method):
    """tol = shift_tol = 1e-14, L = 4 shifts including 0: X, b.grad, sigma.grad and vals.grad within 1e-9 relative of
    np.linalg.solve"""
    B.set_options(tol=1e-14, max_iter=3000, shift_tol=1e-14, shift_max_iter=3000)
    n, ptr, col, val = small_csr(B, case)
    assert n <= 600
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(17)
        b, w = rng.standard_normal(n), rng.standard_normal((SIGMA.size, n))
        vals = _perturbed(val, 1)
        x, gb, gs, gv = _shifted_grads(B, dm, method, b, SIGMA, vals, w)
        A = _dense(n, ptr, col, vals)
        xd = np.stack([np.linalg.solve(A + s * np.eye(n), b) for s in SIGMA])
        lam = np.stack([np.linalg.solve(A.T + s * np.eye(n), w[j]) for j, s in enumerate(SIGMA)])
        rows = np.repeat(np.arange(n), np.diff(ptr))
        want = (xd, lam.sum(axis=0), -np.einsum("ji,ji->j", lam, xd), -(lam[:, rows] * xd[:, col]).sum(axis=0))
        ratios = [np.abs(g.cpu().numpy() - d).max() / np.abs(d).max() for g, d in zip((x, gb, gs, gv), want)]
        print(f"dense {case} {method}: relative deviation X {ratios[0]:.2e}, grad_b {ratios[1]:.2e}, grad_sigma "
              f"{ratios[2]:.2e}, grad_vals {ratios[3]:.2e}")
        assert max(ratios) <= 1e-9, (case, method, ratios)
    finally:
        dm.destroy()


def test_gradcheck(B):
    """torch.autograd.gradcheck (fast mode) on convdiff g = 8, L = 3: the shifted solve in b, sigma and the values, and the
    shifted multiply in x, the values and sigma"""
    torch = _torch()
    B.set_options(tol=1e-15, max_iter=3000, shift_tol=1e-15, shift_max_iter=3000)
    blk = B.gen_block("convdiff", 8, 2.0)
    n = blk.n
    dm = B.DeviceMatrix(blk)
    try:
        vals = blk.diag_arrays()[0].copy()
        rng = np.random.default_rng(2)
        b, s, tv = _cuda(rng.standard_normal(n), True), _cuda(np.array([0.0, 0.5, 2.0]), True), _cuda(vals, True)
        assert torch.autograd.gradcheck(lambda bb, ss, vv: B.shifted_solve_autograd(dm, bb, ss, diag_val=vv), (b, s, tv),
                                        fast_mode=True, atol=1e-6, rtol=1e-4)
        x = _cuda(rng.standard_normal((3, n)), True)
        assert torch.autograd.gradcheck(lambda xx, vv, ss: B.multiply_autograd(dm, xx, diag_val=vv, sigma=ss), (x, tv, s),
                                        fast_mode=True)
    finally:
        dm.destroy()


def test_multiply_with_sigma_backward(B):
    """with sigma: y, grad_x, grad_sigma and grad_vals equal multiply(sigma), the shifted multiply on A^T, dots_async(g, x) and
    value_grad(g, x, 1), bit for bit; without it, nothing changes"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "random")
    rng = np.random.default_rng(4)
    x, w, vals, sig = rng.standard_normal((3, n)), rng.standard_normal((3, n)), _perturbed(val, 3), np.array([0.0, 0.75, -2.5])
    dm, dm2 = _handle(B, n, ptr, col, val), _handle(B, n, ptr, col, val)
    mt2 = dm2.transpose()
    try:
        tx, tv, ts = _cuda(x, True), _cuda(vals, True), _cuda(sig, True)
        y = B.multiply_autograd(dm, tx, diag_val=tv, sigma=ts)
        (y * _cuda(w)).sum().backward()
        dm2.set_values(vals)
        mt2.transpose_values(dm2)
        assert _bits(y) == _bits(dm2.multiply(x, sigma=sig))
        assert _bits(tx.grad) == _bits(mt2.multiply(w, sigma=sig))
        assert _bits(tv.grad) == _bits(dm2.value_grad(w, x, alpha=1.0)[0])
        assert _bits(ts.grad) == _bits(dm2.dots_async(_cuda(w), _cuda(x)))
        tx2, tv2 = _cuda(x, True), _cuda(vals, True)
        y2 = B.multiply_autograd(dm, tx2, diag_val=tv2)
        (y2 * _cuda(w)).sum().backward()
        assert _bits(y2) == _bits(dm2.multiply(x)) and _bits(tx2.grad) == _bits(mt2.multiply(w))
    finally:
        for d in (dm, dm2):
            d.destroy()


@pytest.mark.parametrize("mega", [0, 1, 2])
@pytest.mark.parametrize("method", ["shifted_lopbicg_switching", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab",
                                    "shifted_lopbicg"])
def test_equals_explicit_sequence(B, method, mega):
    """X equals shifted_solve_async on a second handle; every lambda_j = refresh -> shift_diagonal_async -> solve_async equals a
    solve on a fresh handle of host-shifted transposed blocks; b.grad is numpy's left-to-right sum of the lambda_j, sigma.grad
    -dots_async(lambda, X) and vals.grad value_grad_async(lambda, X, -1), bit for bit"""
    torch = _torch()
    B.set_options(mega=mega)
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(3)
    L = SIGMA.size
    b, w, vals = rng.standard_normal(n), rng.standard_normal((L, n)), _perturbed(val, 2)
    dm, dm2 = _handle(B, n, ptr, col, val), _handle(B, n, ptr, col, val)
    mt2 = dm2.transpose()
    tp, tc, tv = transposed_csr(n, ptr, col, vals)
    try:
        x, gb, gs, gv = _shifted_grads(B, dm, method, b, SIGMA, vals, w, seed=1)
        dm2.set_values_async(_cuda(vals))
        ts = _cuda(SIGMA)
        x2, r2 = torch.zeros(L, n, dtype=torch.float64, device="cuda"), _cuda(b)
        dm2.shifted_solve_async(method, x2, r2, ts, 1)
        lam = torch.zeros(L, n, dtype=torch.float64, device="cuda")
        for j in range(L):
            mt2.transpose_values_async(dm2)
            mt2.shift_diagonal_async(ts[j:j + 1])
            mt2.solve_async("bicgstab", lam[j], _cuda(w[j]))
        gs2 = dm2.dots_async(lam, x2)
        gv2, _ = dm2.value_grad_async(lam, x2, alpha=-1.0)
        torch.cuda.synchronize()
        assert _bits(x) == _bits(x2), (method, mega)
        lam_np = lam.cpu().numpy()
        acc = lam_np[0].copy()
        for j in range(1, L):
            acc = acc + lam_np[j]
        assert _bits(gb) == _bits(acc), (method, mega)
        assert _bits(gs) == _bits(-gs2), (method, mega)
        assert _bits(gv) == _bits(gv2), (method, mega)
        for j in range(L):
            fresh = _host_shifted(B, n, tp, tc, tv, [SIGMA[j]])
            try:
                lf = torch.zeros(n, dtype=torch.float64, device="cuda")
                fresh.solve_async("bicgstab", lf, _cuda(w[j]))
                torch.cuda.synchronize()
                assert _bits(lf) == _bits(lam[j]), (method, mega, j)
            finally:
                fresh.destroy()
    finally:
        for d in (dm, dm2):
            d.destroy()


# ---- shift_diagonal_async -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["convdiff", "random", "tprime", "golden"])
def test_shift_on_transpose_equals_host_shifted_transpose(B, case):
    """after transpose_values_async(A) and shift_diagonal_async(sigma), every result on the transpose (spmv, a shifted
    multiply, every method and every shifted method) is bit-identical to a handle of host-shifted transposed blocks; the same
    holds for A itself"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, case)
    tp, tc, tv = transposed_csr(n, ptr, col, val)
    if not (_has_diagonal(n, ptr, col) and _has_diagonal(n, tp, tc)):
        pytest.skip(f"{case}: a row without a diagonal entry")
    dm = _handle(B, n, ptr, col, val)
    mt = dm.transpose()
    sig = _cuda(np.array([0.75]))
    try:
        mt.transpose_values_async(dm)
        mt.shift_diagonal_async(sig)
        dm.shift_diagonal_async(sig)
        torch.cuda.synchronize()
        for h, (p, c, v) in ((mt, (tp, tc, tv)), (dm, (ptr, col, val))):
            fresh = _host_shifted(B, n, p, c, v, [0.75])
            try:
                _same_everywhere(B, h, fresh, n, (case, "transpose" if h is mt else "A"))
            finally:
                fresh.destroy()
    finally:
        for d in (mt, dm):
            d.destroy()


def test_shifts_accumulate_like_the_synchronous_shift(B):
    """shift_diagonal_async(0.75), then (-0.125): the same bits as shift_diagonal(0.75), shift_diagonal(-0.125) and a fresh
    handle of host-shifted blocks"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "tprime")
    dm, dm2 = _handle(B, n, ptr, col, val), _handle(B, n, ptr, col, val)
    fresh = _host_shifted(B, n, ptr, col, val, [0.75, -0.125])
    try:
        s = _cuda(np.array([0.75, -0.125]))
        dm.shift_diagonal_async(s[0:1])
        dm.shift_diagonal_async(s[1:2])
        dm2.shift_diagonal(0.75)
        dm2.shift_diagonal(-0.125)
        torch.cuda.synchronize()
        x = np.random.default_rng(1).standard_normal(n)
        assert _bits(dm.spmv(x)) == _bits(dm2.spmv(x)) == _bits(fresh.spmv(x))
        _same_everywhere(B, dm, fresh, n, "accumulated")
    finally:
        for d in (dm, dm2, fresh):
            d.destroy()


def test_shift_without_a_diagonal_entry_changes_nothing(B):
    """the hand-made 7 x 7 matrix (row 6 of A has no diagonal entry, row 6 of A^T is empty): -1 / ValueError and unchanged
    values, on A and on its transpose; prepare_shifted_autograd refuses it"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "handmade")
    dm = _handle(B, n, ptr, col, val)
    mt = dm.transpose()
    try:
        mt.transpose_values(dm)
        x = np.random.default_rng(2).standard_normal(n)
        before = [_bits(dm.spmv(x)), _bits(mt.spmv(x))]
        sig = _cuda(np.array([1.0]))
        for h in (dm, mt):
            with pytest.raises(ValueError, match="no diagonal entry"):
                h.shift_diagonal_async(sig)
            assert B.lib.bicg_matrix_shift_diagonal_async(h.h, C.c_void_p(sig.data_ptr()), None) == -1
            assert B.lib.bicg_matrix_shift_diagonal_async_prepare(h.h) == -1
        torch.cuda.synchronize()
        assert [_bits(dm.spmv(x)), _bits(mt.spmv(x))] == before
        with pytest.raises(ValueError, match="diagonal entry"):
            dm.prepare_shifted_autograd("shifted_lopbicgstab", 2)
    finally:
        for d in (mt, dm):
            d.destroy()


def test_shift_capture_needs_prepare_and_replays_new_sigma(B):
    """inside a capture before prepare: -2 (RuntimeError naming the prepare); after it, a captured shift replayed with a new
    sigma in its buffer adds that value: replays of 0.5 then -0.25 equal host shifts by both in turn"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    try:
        buf = _cuda(np.array([0.5]))
        x = _cuda(np.ones(n))
        dm.multiply_async(x, torch.empty_like(x))                 # the handle's first asynchronous use, outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match="prepare_shift_diagonal_async"):
            with torch.cuda.graph(g):
                dm.shift_diagonal_async(buf)
        del g
        torch.cuda.synchronize()
        dm.prepare_shift_diagonal_async()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            dm.shift_diagonal_async(buf)
        xs = np.random.default_rng(3).standard_normal(n)
        shifts = []
        for s in (0.5, -0.25):
            with torch.no_grad():
                buf.fill_(s)
            g.replay()
            torch.cuda.synchronize()
            shifts.append(s)
            fresh = _host_shifted(B, n, ptr, col, val, shifts)
            try:
                assert _bits(dm.spmv(xs)) == _bits(fresh.spmv(xs)), shifts
            finally:
                fresh.destroy()
        del g
    finally:
        dm.destroy()


# ---- dots_async -----------------------------------------------------------------------------------------------------------
def dots_model(u, v):
    """out[j] of one rank in the order include/bicgstab_b200.h pins: fma chains over chunks of 4096 (thread t: elements
    t + 256 s), the tree over 256 threads, chunk sums added in chunk order onto +0.0"""
    out = []
    for uj, vj in zip(u, v):
        n = uj.size
        nch = (n + 4095) // 4096
        pad = nch * 4096
        up, vp = np.zeros(pad), np.zeros(pad)
        up[:n], vp[:n] = uj, vj
        valid = np.arange(pad) < n
        uc, vc, mc = (a.reshape(nch, 16, 256) for a in (up, vp, valid))
        p = np.zeros((nch, 256))
        for s in range(16):
            p = np.where(mc[:, s], fma(uc[:, s], vc[:, s], p), p)
        h = 128
        while h:
            p[:, :h] = p[:, :h] + p[:, h:2 * h]
            h //= 2
        tot = 0.0
        for c in range(nch):
            tot = tot + p[c, 0]
        out.append(tot)
    return np.array(out)


def _dots_inputs(nvec, n, seed):
    rng = np.random.default_rng(seed)
    u = rng.standard_normal((nvec, n)) * np.exp2(rng.integers(-40, 40, (nvec, n)))
    v = rng.standard_normal((nvec, n)) * np.exp2(rng.integers(-40, 40, (nvec, n)))
    u[:, ::7] = 0.0
    v[:, 3::11] = -0.0
    u[0, ::5] = -u[0, ::5]
    if nvec > 1:
        u[1], v[1] = -0.0, 1.0                                   # every product -0: the sum is +0
    if nvec > 2:
        v[2] = u[2]
        u[2, 1::2] = -u[2, ::2][:u[2, 1::2].size]                # pairs that cancel exactly
        v[2, 1::2] = v[2, ::2][:v[2, 1::2].size]
    return u, v


@pytest.mark.parametrize("n", [1, 255, 257, 4095, 4096, 4097, 3 * 4096 + 5, 512 * 4096 + 4097])
def test_dots_against_cpu_model(B, n):
    """nvec = 1, 3, 8, 9, 17 on n_loc either side of the chunk (4096) and tile (512 chunks) sizes, with signed zeros and exact
    cancellations: bit for bit the CPU model; the same bits on every run and every replay of a captured call"""
    torch = _torch()
    import scipy.sparse as sp
    A = sp.identity(n, format="csr")
    dm = _handle(B, n, A.indptr, A.indices, A.data)
    try:
        for nvec in (1, 3, 8, 9, 17):
            if n > 100000 and nvec not in (1, 9):
                continue
            u, v = _dots_inputs(nvec, n, nvec * 1000 + n % 997)
            want = dots_model(u, v)
            tu, tv = _cuda(u), _cuda(v)
            got = dm.dots_async(tu, tv)
            again = dm.dots_async(tu, tv)
            torch.cuda.synchronize()
            assert _bits(got) == _bits(want), (n, nvec, got.cpu().numpy(), want)
            assert _bits(again) == _bits(want), (n, nvec)
            if nvec > 1:
                assert not np.signbit(got[1].item()) and got[1].item() == 0.0, (n, nvec)
        u, v = _dots_inputs(3, n, 5)
        tu, tv = _cuda(u), _cuda(v)
        out = torch.full((3,), np.nan, dtype=torch.float64, device="cuda")
        one = dm.dots_async(tu[0], tv[0])
        torch.cuda.synchronize()
        assert _bits(one) == _bits(dots_model(u[:1], v[:1])), n
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            dm.dots_async(tu, tv, out=out)
        for k in range(2):
            u2, v2 = _dots_inputs(3, n, 50 + k)
            with torch.no_grad():
                tu.copy_(torch.from_numpy(u2))
                tv.copy_(torch.from_numpy(v2))
            g.replay()
            torch.cuda.synchronize()
            assert _bits(out) == _bits(dots_model(u2, v2)), (n, k)
        del g
    finally:
        dm.destroy()


# ---- behaviour ------------------------------------------------------------------------------------------------------------
def test_partial_loss_and_records(B):
    """a loss over shift 1 only: lambda_j = 0 for the others with no iterations (adjoint_result), their sigma.grad is 0, and
    b.grad is lambda_1; the forward's bicg_shift_result and every converged adjoint solve are recorded"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    L = SIGMA.size
    rng = np.random.default_rng(11)
    b, vals = rng.standard_normal(n), _perturbed(val, 4)
    w = np.zeros((L, n))
    w[1] = rng.standard_normal(n)
    dm = _handle(B, n, ptr, col, val)
    try:
        res = torch.zeros(32, dtype=torch.uint8, device="cuda")
        ares = torch.zeros(L * 24, dtype=torch.uint8, device="cuda")
        x, gb, gs, gv = _shifted_grads(B, dm, "shifted_lopbicgstab", b, SIGMA, vals, w, result=res, adjoint_result=ares)
        rec = B.decode_shift_result(res)
        assert rec["converged"] and rec["error"] == 0 and rec["iters"] > 0, rec
        gs = gs.cpu().numpy()
        for j in range(L):
            a = B.decode_result(ares[24 * j:24 * (j + 1)])
            assert a["error"] == 0, (j, a)
            if j == 1:
                assert a["converged"] and a["iters"] > 0, a
            else:
                assert a["iters"] == 0 and gs[j] == 0.0, (j, a, gs[j])
        assert not np.isnan(gb.cpu().numpy()).any() and not np.isnan(gv.cpu().numpy()).any()
        # lambda_1 alone: b.grad of the same loss with L = 1 (the same refresh, shift and solve; the zero lambda_j add nothing)
        _, gb1, _, _ = _shifted_grads(B, dm, "shifted_lopbicgstab", b, SIGMA[1:2], vals, w[1:2])
        assert np.array_equal(gb.cpu().numpy(), gb1.cpu().numpy())
    finally:
        dm.destroy()


def test_stale_handle_and_interleaved_forwards(B):
    """forward with v1, set_values(v2), backward: v1's gradients; two forwards with different values and shifts, one backward:
    each term's gradients equal those computed alone"""
    n, ptr, col, val = _case_csr(B, "tprime")
    rng = np.random.default_rng(5)
    L = 3
    b1, b2 = rng.standard_normal(n), rng.standard_normal(n)
    w1, w2 = rng.standard_normal((L, n)), rng.standard_normal((L, n))
    s1, s2 = SIGMA[:L], SIGMA[1:L + 1]
    v1, v2 = _perturbed(val, 1), _perturbed(val, 4)
    dm = _handle(B, n, ptr, col, val)
    try:
        alone1 = [_bits(a) for a in _shifted_grads(B, dm, "shifted_pipe_lopbicgstab", b1, s1, v1, w1)]
        alone2 = [_bits(a) for a in _shifted_grads(B, dm, "shifted_pipe_lopbicgstab", b2, s2, v2, w2)]
        tb, ts, tv = _cuda(b1, True), _cuda(s1, True), _cuda(v1, True)
        x = B.shifted_solve_autograd(dm, tb, ts, "shifted_pipe_lopbicgstab", diag_val=tv)
        dm.set_values(v2)
        (x * _cuda(w1)).sum().backward()
        assert [_bits(a) for a in (x, tb.grad, ts.grad, tv.grad)] == alone1
        t1 = [_cuda(a, True) for a in (b1, s1, v1)]
        t2 = [_cuda(a, True) for a in (b2, s2, v2)]
        x1 = B.shifted_solve_autograd(dm, t1[0], t1[1], "shifted_pipe_lopbicgstab", diag_val=t1[2])
        x2 = B.shifted_solve_autograd(dm, t2[0], t2[1], "shifted_pipe_lopbicgstab", diag_val=t2[2])
        ((x1 * _cuda(w1)).sum() + (x2 * _cuda(w2)).sum()).backward()
        assert [_bits(a) for a in [x1] + [t.grad for t in t1]] == alone1
        assert [_bits(a) for a in [x2] + [t.grad for t in t2]] == alone2
    finally:
        dm.destroy()


def test_side_stream(B):
    """forward and backward on a side stream with no host synchronisation equal the default-stream run"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(9)
    b, w, vals = rng.standard_normal(n), rng.standard_normal((SIGMA.size, n)), _perturbed(val, 6)
    dm = _handle(B, n, ptr, col, val)
    try:
        want = [_bits(a) for a in _shifted_grads(B, dm, "shifted_lopbicg", b, SIGMA, vals, w)]
        tb, ts, tv, tw = _cuda(b, True), _cuda(SIGMA, True), _cuda(vals, True), _cuda(w)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            x = B.shifted_solve_autograd(dm, tb, ts, "shifted_lopbicg", diag_val=tv)
            (x * tw).sum().backward()
        s.synchronize()
        assert [_bits(a) for a in (x, tb.grad, ts.grad, tv.grad)] == want
    finally:
        dm.destroy()


def test_graph_capture_replay(B):
    """forward + loss.backward() captured in torch.cuda.graph after prepare_shifted_autograd, replayed with three
    (b, sigma, values) sets: bit-identical to uncaptured runs; without the prepare the capture raises and names it"""
    torch = _torch()
    method = "shifted_lopbicgstab"
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(10)
    L = SIGMA.size
    sets = [(rng.standard_normal(n), SIGMA * (1.0 + k / 8.0), _perturbed(val, k)) for k in (1, 2, 3)]
    w = rng.standard_normal((L, n))
    dm = _handle(B, n, ptr, col, val)
    try:
        dm.prepare_shifted_autograd(method, L)
        tb, ts, tv, tw = _cuda(sets[0][0], True), _cuda(sets[0][1], True), _cuda(sets[0][2], True), _cuda(w)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                               # warm-up, as torch's whole-network capture asks
            x = B.shifted_solve_autograd(dm, tb, ts, method, diag_val=tv)
            (x * tw).sum().backward()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        tb.grad = ts.grad = tv.grad = None
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            xs = B.shifted_solve_autograd(dm, tb, ts, method, diag_val=tv)
            (xs * tw).sum().backward()
        for bv, sv, vv in sets:
            with torch.no_grad():
                tb.copy_(torch.from_numpy(bv))
                ts.copy_(torch.from_numpy(sv))
                tv.copy_(torch.from_numpy(vv))
            g.replay()
            torch.cuda.synchronize()
            got = [_bits(a) for a in (xs, tb.grad, ts.grad, tv.grad)]
            want = [_bits(a) for a in _shifted_grads(B, dm, method, bv, sv, vv, w)]
            assert got == want
        del g
    finally:
        dm.destroy()
    for prepared in (False, True):              # nothing prepared: the forward raises; the forward alone: the backward does
        dm = _handle(B, n, ptr, col, val)
        try:
            if prepared:
                dm.prepare_shifted_async(method, L)
            tb, ts, tw = _cuda(sets[0][0], True), _cuda(sets[0][1], True), _cuda(w)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with pytest.raises(RuntimeError, match="prepare_shifted_autograd"):
                with torch.cuda.graph(g):
                    x = B.shifted_solve_autograd(dm, tb, ts, method)
                    (x * tw).sum().backward()
            del g
            torch.cuda.synchronize()
        finally:
            dm.destroy()


def test_errors(B):
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    b = torch.ones(n, dtype=torch.float64, device="cuda")
    s = torch.zeros(3, dtype=torch.float64, device="cuda")
    try:
        with pytest.raises(ValueError, match="1-d"):
            B.shifted_solve_autograd(dm, b, s.view(1, 3))
        with pytest.raises(ValueError, match="seed"):
            B.shifted_solve_autograd(dm, b, s, seed=3)
        with pytest.raises(ValueError, match="seed"):
            B.shifted_solve_autograd(dm, b, s, seed=-1)
        with pytest.raises(ValueError, match="without diag_val"):
            B.shifted_solve_autograd(dm, b, s, offd_val=torch.ones(3, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="shape"):
            B.shifted_solve_autograd(dm, b, s, x0=torch.zeros(2, n, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="adjoint_result"):
            B.shifted_solve_autograd(dm, b, s, adjoint_result=torch.zeros(24, dtype=torch.uint8, device="cuda"))
        with pytest.raises(ValueError, match="shape"):
            B.multiply_autograd(dm, torch.ones(2, n, dtype=torch.float64, device="cuda"), sigma=s)
        with pytest.raises(ValueError, match="shape"):
            dm.dots_async(b, torch.ones(2, n, dtype=torch.float64, device="cuda"))
    finally:
        dm.destroy()
