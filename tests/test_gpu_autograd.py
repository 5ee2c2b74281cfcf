"""GPU: loss.backward() through solves and products on a resident matrix (solve_autograd, multiply_autograd).  The backward of
x = A^-1 b solves A^T lambda = dL/dx on the handle's transpose and forms dL/da_e = -lambda_i x_c with the value-gradient kernel.
Checked: against dense numpy, with torch.autograd.gradcheck, bit for bit against the explicit sequence refresh -> solve on A^T
-> value_grad on every method and loop path, for stale handles, interleaved forwards, zero output gradients, several
right-hand sides, side streams and CUDA graph replays, and for the convergence records and argument errors."""
import numpy as np
import pytest

from helpers import METHODS
from test_gpu_transpose import _case_csr, transposed_csr
from test_gpu_value_grad import replica

pytestmark = pytest.mark.gpu

RATIOS = []          # the largest relative deviation from dense numpy seen, per quantity (printed by the dense test)


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, tol=1e-10, max_iter=1000, mega=1, resident=1)
    yield
    B.set_options(tol=1e-15, max_iter=1000, mega=1, resident=1)


def _torch():
    import torch
    return torch


def _bits(a):
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def small_csr(B, case):
    """(n, ptr, col, val) with n <= 600: convection-diffusion, the golden shifted matrix, T' at g = 8 with row-scaled values"""
    if case == "tprime8":
        blk = B.gen_block("stencil15", 8, 14.0)
        ptr, col, val = (np.asarray(a) for a in B.block_to_global_csr(blk))
        val = val * (1.0 + (np.repeat(np.arange(blk.n), np.diff(ptr)) % 5) / 16.0)
        return blk.n, ptr.astype(np.int64), col.astype(np.int64), val.astype(np.float64)
    return _case_csr(B, case)


def _handle(B, n, ptr, col, val):
    return B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))


def _cuda(a, grad=False):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(grad)


def _perturbed(v, k):
    return v * (1.0 + ((np.arange(v.size) * (2 * k + 1) + k) % 7) / 64.0)


def _solve_grads(B, dm, method, b, vals, w, **kw):
    """x, b.grad and vals.grad of loss = (w * x).sum() with x = solve_autograd(dm, b, method, diag_val=vals)"""
    tb, tv = _cuda(b, True), _cuda(vals, True)
    x = B.solve_autograd(dm, tb, method, diag_val=tv, **kw)
    (x * _cuda(w)).sum().backward()
    return x.detach(), tb.grad, tv.grad


@pytest.mark.parametrize("case", ["convdiff", "golden", "tprime8"])
def test_against_dense_numpy(B, case):
    """tol = 1e-14: b.grad = A^-T w and vals.grad_e = -lambda_i x_c, within 1e-9 relative of np.linalg.solve"""
    B.set_options(tol=1e-14, max_iter=3000)
    n, ptr, col, val = small_csr(B, case)
    assert n <= 600
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(7)
        b, w = rng.standard_normal(n), rng.standard_normal(n)
        vals = _perturbed(val, 1)
        x, gb, gv = _solve_grads(B, dm, "bicgstab", b, vals, w)
        A = np.zeros((n, n))
        np.add.at(A, (np.repeat(np.arange(n), np.diff(ptr)), col), vals)
        xd, lam = np.linalg.solve(A, b), np.linalg.solve(A.T, w)
        rows = np.repeat(np.arange(n), np.diff(ptr))
        gvd = -lam[rows] * xd[col]
        ratios = [np.abs(got.cpu().numpy() - want).max() / np.abs(want).max() for got, want in ((x, xd), (gb, lam), (gv, gvd))]
        RATIOS.append((case, ratios))
        print(f"dense {case}: relative deviation x {ratios[0]:.2e}, grad_b {ratios[1]:.2e}, grad_vals {ratios[2]:.2e}")
        assert max(ratios) <= 1e-9, (case, ratios)
    finally:
        dm.destroy()


def test_gradcheck(B):
    """torch.autograd.gradcheck (fast mode) on convdiff g = 8 in b and the values, for the solve and for the multiply"""
    torch = _torch()
    B.set_options(tol=1e-15, max_iter=3000)
    blk = B.gen_block("convdiff", 8, 2.0)
    n = blk.n
    dm = B.DeviceMatrix(blk)
    try:
        vals = blk.diag_arrays()[0].copy()
        b, tv = _cuda(np.random.default_rng(1).standard_normal(n), True), _cuda(vals, True)
        assert torch.autograd.gradcheck(lambda bb, vv: B.solve_autograd(dm, bb, diag_val=vv), (b, tv), fast_mode=True,
                                        atol=1e-6, rtol=1e-4)
        assert torch.autograd.gradcheck(lambda xx, vv: B.multiply_autograd(dm, xx, diag_val=vv), (b, tv), fast_mode=True)
    finally:
        dm.destroy()


@pytest.mark.parametrize("mega", [0, 1, 2])
@pytest.mark.parametrize("method", METHODS)
def test_equals_explicit_sequence(B, method, mega):
    """x, b.grad and vals.grad equal set_values -> solve -> refresh A^T -> solve on A^T from 0 -> value_grad(lambda, x, -1), bit
    for bit; b.grad equals a solve on a handle freshly created from the transposed blocks"""
    torch = _torch()
    B.set_options(mega=mega)
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(3)
    b, w, vals = rng.standard_normal(n), rng.standard_normal(n), _perturbed(val, 2)
    dm, dm2 = _handle(B, n, ptr, col, val), _handle(B, n, ptr, col, val)
    mt2 = dm2.transpose()
    tp, tc, tv = transposed_csr(n, ptr, col, vals)
    fresh = _handle(B, n, tp, tc, tv)
    try:
        x, gb, gv = _solve_grads(B, dm, method, b, vals, w)
        dm2.set_values_async(_cuda(vals))
        x2, r2 = torch.zeros(n, dtype=torch.float64, device="cuda"), _cuda(b)
        dm2.solve_async(method, x2, r2)
        mt2.transpose_values_async(dm2)
        lam, rl = torch.zeros(n, dtype=torch.float64, device="cuda"), _cuda(w)
        mt2.solve_async(method, lam, rl)
        gv2, _ = dm2.value_grad_async(lam, x2, alpha=-1.0)
        lf, rf = torch.zeros(n, dtype=torch.float64, device="cuda"), _cuda(w)
        fresh.solve_async(method, lf, rf)
        torch.cuda.synchronize()
        assert _bits(x) == _bits(x2), (method, mega)
        assert _bits(gb) == _bits(lam) == _bits(lf), (method, mega)
        assert _bits(gv) == _bits(gv2), (method, mega)
    finally:
        for d in (dm, dm2, fresh):
            d.destroy()


def test_multiply_backward(B):
    """grad_x is the multiply on A^T bit for bit, grad_vals is value_grad(grad_y, x, 1)"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "random")
    rng = np.random.default_rng(4)
    x, w, vals = rng.standard_normal((2, n)), rng.standard_normal((2, n)), _perturbed(val, 3)
    dm, dm2 = _handle(B, n, ptr, col, val), _handle(B, n, ptr, col, val)
    mt2 = dm2.transpose()
    try:
        tx, tv = _cuda(x, True), _cuda(vals, True)
        y = B.multiply_autograd(dm, tx, diag_val=tv)
        (y * _cuda(w)).sum().backward()
        dm2.set_values(vals)
        mt2.transpose_values(dm2)
        assert _bits(y) == _bits(dm2.multiply(x))
        assert _bits(tx.grad) == _bits(mt2.multiply(w))
        assert _bits(tv.grad) == _bits(dm2.value_grad(w, x, alpha=1.0)[0])
        # values-only gradients: the backward leaves the handle's values alone (the value gradient needs the pattern only)
        tv2 = _cuda(vals, True)
        y = B.multiply_autograd(dm, _cuda(x), diag_val=tv2)
        dm.set_values(val)
        (y * _cuda(w)).sum().backward()
        assert _bits(tv2.grad) == _bits(dm2.value_grad(w, x, alpha=1.0)[0])
        dm2.set_values(val)
        assert _bits(dm.multiply(x)) == _bits(dm2.multiply(x))
    finally:
        for d in (dm, dm2):
            d.destroy()


def test_stale_handle_and_interleaved_forwards(B):
    """forward with v1, set_values(v2), backward: v1's gradients; two forwards with different values, one backward: each term's
    gradients equal those computed alone"""
    n, ptr, col, val = _case_csr(B, "tprime")
    rng = np.random.default_rng(5)
    b1, b2, w1, w2 = (rng.standard_normal(n) for _ in range(4))
    v1, v2 = _perturbed(val, 1), _perturbed(val, 4)
    dm = _handle(B, n, ptr, col, val)
    try:
        alone1 = _solve_grads(B, dm, "bicgstab", b1, v1, w1)
        alone2 = _solve_grads(B, dm, "bicgstab", b2, v2, w2)
        tb, tv = _cuda(b1, True), _cuda(v1, True)
        x = B.solve_autograd(dm, tb, diag_val=tv)
        dm.set_values(v2)
        (x * _cuda(w1)).sum().backward()
        assert [_bits(x), _bits(tb.grad), _bits(tv.grad)] == [_bits(a) for a in alone1]
        tb1, tv1, tb2, tv2 = _cuda(b1, True), _cuda(v1, True), _cuda(b2, True), _cuda(v2, True)
        x1 = B.solve_autograd(dm, tb1, diag_val=tv1)
        x2 = B.solve_autograd(dm, tb2, diag_val=tv2)
        ((x1 * _cuda(w1)).sum() + (x2 * _cuda(w2)).sum()).backward()
        assert [_bits(x1), _bits(tb1.grad), _bits(tv1.grad)] == [_bits(a) for a in alone1]
        assert [_bits(x2), _bits(tb2.grad), _bits(tv2.grad)] == [_bits(a) for a in alone2]
    finally:
        dm.destroy()


@pytest.mark.parametrize("mega", [0, 1, 2])
def test_zero_grad_output(B, mega):
    """a zero dL/dx gives zero gradients and no NaN on every method"""
    B.set_options(mega=mega)
    n, ptr, col, val = _case_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    try:
        for method in METHODS:
            rng = np.random.default_rng(6)
            _, gb, gv = _solve_grads(B, dm, method, rng.standard_normal(n), _perturbed(val, 1), np.zeros(n))
            for g in (gb, gv):
                g = g.cpu().numpy()
                assert not np.isnan(g).any() and not np.any(g), (method, mega)
    finally:
        dm.destroy()


@pytest.mark.parametrize("k", [3, 9])
def test_several_right_hand_sides(B, k):
    """b of shape (k, n): x and b.grad rows equal single-vector runs; vals.grad (one value gradient over k vectors, crossing
    a batch at k = 9) equals the replica on b.grad and x"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(8)
    b, w, vals = rng.standard_normal((k, n)), rng.standard_normal((k, n)), _perturbed(val, 5)
    dm = _handle(B, n, ptr, col, val)
    try:
        res, ares = torch.zeros(k * 24, dtype=torch.uint8, device="cuda"), torch.zeros(k * 24, dtype=torch.uint8, device="cuda")
        x, gb, gv = _solve_grads(B, dm, "bicgstab", b, vals, w, result=res, adjoint_result=ares)
        for j in range(k):
            xj, gbj, _ = _solve_grads(B, dm, "bicgstab", b[j], vals, w[j])
            assert _bits(x[j]) == _bits(xj) and _bits(gb[j]) == _bits(gbj), (k, j)
        for t in (res, ares):
            for j in range(k):
                rec = B.decode_result(t[24 * j:24 * (j + 1)])
                assert rec["converged"] and rec["error"] == 0 and rec["iters"] > 0, (k, j, rec)
        rows = np.repeat(np.arange(n), np.diff(ptr))
        idx = np.arange(int(ptr[-1]))
        want = replica(rows[idx], col[idx], gb.cpu().numpy(), x.cpu().numpy(), -1.0, 0.0, None)
        assert _bits(gv.cpu().numpy()[idx]) == _bits(want), k
    finally:
        dm.destroy()


def test_transposed_loss_with_several_right_hand_sides(B):
    """b of shape (k, n) and a loss over x.T: torch hands the backward a gradient with column-major strides; the gradients equal
    those of the same loss written over x, bit for bit"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(12)
    k = 3
    b, w, vals = rng.standard_normal((k, n)), rng.standard_normal((n, k)), _perturbed(val, 7)
    dm = _handle(B, n, ptr, col, val)
    try:
        got = []
        for transposed in (True, False):
            tb, tv, tw = _cuda(b, True), _cuda(vals, True), _cuda(w)
            x = B.solve_autograd(dm, tb, diag_val=tv)
            loss = (x.T * tw).sum() if transposed else (x * tw.T.contiguous()).sum()
            loss.backward()
            got.append([_bits(x), _bits(tb.grad), _bits(tv.grad)])
        assert got[0] == got[1]
    finally:
        dm.destroy()


def test_side_stream(B):
    """forward and backward on a side stream with no host synchronisation equal the default-stream run"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(9)
    b, w, vals = rng.standard_normal(n), rng.standard_normal(n), _perturbed(val, 6)
    dm = _handle(B, n, ptr, col, val)
    try:
        want = [_bits(a) for a in _solve_grads(B, dm, "pipe_bicgstab", b, vals, w)]
        tb, tv, tw = _cuda(b, True), _cuda(vals, True), _cuda(w)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            x = B.solve_autograd(dm, tb, "pipe_bicgstab", diag_val=tv)
            (x * tw).sum().backward()
        s.synchronize()
        assert [_bits(x), _bits(tb.grad), _bits(tv.grad)] == want
    finally:
        dm.destroy()


def test_graph_capture_replay(B):
    """forward + loss.backward() captured in torch.cuda.graph after prepare_autograd, replayed with three (b, values) sets:
    bit-identical to eager runs; the same capture without prepare_autograd raises"""
    torch = _torch()
    method = "bicgstab"
    n, ptr, col, val = _case_csr(B, "convdiff")
    rng = np.random.default_rng(10)
    sets = [(rng.standard_normal(n), _perturbed(val, k)) for k in (1, 2, 3)]
    w = rng.standard_normal(n)
    dm = _handle(B, n, ptr, col, val)
    try:
        dm.prepare_autograd(method)
        tb, tv, tw = _cuda(sets[0][0], True), _cuda(sets[0][1], True), _cuda(w)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                               # warm-up, as torch's whole-network capture asks
            x = B.solve_autograd(dm, tb, method, diag_val=tv)
            (x * tw).sum().backward()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        tb.grad, tv.grad = None, None
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            xs = B.solve_autograd(dm, tb, method, diag_val=tv)
            (xs * tw).sum().backward()
        for bv, vv in sets:
            with torch.no_grad():
                tb.copy_(torch.from_numpy(bv))
                tv.copy_(torch.from_numpy(vv))
            g.replay()
            torch.cuda.synchronize()
            got = [_bits(xs), _bits(tb.grad), _bits(tv.grad)]
            want = [_bits(a) for a in _solve_grads(B, dm, method, bv, vv, w)]
            assert got == want
        del g
    finally:
        dm.destroy()
    dm = _handle(B, n, ptr, col, val)
    try:
        dm.prepare_async(method)                                 # the forward can be captured, the backward cannot
        tb, tv = _cuda(sets[0][0], True), _cuda(sets[0][1], True)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match="prepare_autograd"):
            with torch.cuda.graph(g):
                x = B.solve_autograd(dm, tb, method, diag_val=tv)
                (x * tw).sum().backward()
        del g
        torch.cuda.synchronize()
    finally:
        dm.destroy()


def test_errors(B):
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    try:
        with pytest.raises(TypeError, match="CUDA float64 tensor"):
            B.solve_autograd(dm, np.ones(n))
        with pytest.raises(TypeError, match="CUDA float64 tensor"):
            B.multiply_autograd(dm, np.ones(n))
        with pytest.raises(ValueError, match="shape"):
            B.solve_autograd(dm, torch.ones(n + 1, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="shape"):
            B.solve_autograd(dm, torch.ones(2, 3, n, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="shape"):
            B.solve_autograd(dm, torch.ones(n, dtype=torch.float64, device="cuda"), x0=torch.zeros(1, n, dtype=torch.float64,
                                                                                                   device="cuda"))
        with pytest.raises(ValueError, match="diag_val"):
            B.solve_autograd(dm, torch.ones(n, dtype=torch.float64, device="cuda"),
                             diag_val=torch.ones(val.size + 1, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="offd_val"):
            B.solve_autograd(dm, torch.ones(n, dtype=torch.float64, device="cuda"),
                             offd_val=torch.ones(3, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="offd_val"):
            B.multiply_autograd(dm, torch.ones(n, dtype=torch.float64, device="cuda"),
                                offd_val=torch.ones(3, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="result"):
            B.solve_autograd(dm, torch.ones(n, dtype=torch.float64, device="cuda"),
                             result=torch.zeros(23, dtype=torch.uint8, device="cuda"))
    finally:
        dm.destroy()
