"""Differentiable solves, shifted solves and products on a resident matrix (DeviceMatrix), for loss.backward() through them.

    x = solve_autograd(dm, b, "bicgstab", diag_val=vals)              # x = A(vals)^-1 b
    X = shifted_solve_autograd(dm, b, sigma, diag_val=vals)           # X[j] = (A(vals) + sigma_j I)^-1 b
    y = multiply_autograd(dm, x, diag_val=vals, sigma=s)              # y_j = (A(vals) + s_j I) x_j
    loss = f(x, X, y); loss.backward()                                 # b.grad, sigma.grad, s.grad, vals.grad

For x = A^-1 b and a loss L(x), with lambda = A^-T dL/dx: dL/db = lambda and dL/da_e = -lambda_i x_c for every stored entry
e = (i, c).  The backward solves with the handle's transpose (DeviceMatrix.transpose, kept on the handle) after refreshing its
values from the forward's, and forms dL/da with DeviceMatrix.value_grad_async in the block order set_values takes.  For the
shifted solve X_j = (A + sigma_j I)^-1 b, with lambda_j = (A^T + sigma_j I)^-1 dL/dX_j, one adjoint solve per shift on the
transpose refreshed and shifted by sigma_j on the device: dL/db = sum_j lambda_j (in j order), dL/dsigma_j = -<lambda_j, X_j>
(DeviceMatrix.dots_async, summed over every rank), and dL/da_e = -sum_j lambda_j[i] X_j[c] (sigma_j I is no stored value).
For y_j = (A + s_j I) x_j: dL/dx_j = (A^T + s_j I) dL/dy_j and dL/ds_j = <dL/dy_j, x_j>.  Forward and backward are
stream-ordered on torch's current stream, without a host synchronisation, so both can be captured by torch.cuda.graph once
dm.prepare_autograd(method) (dm.prepare_shifted_autograd(method, sigma_len) for shifted solves) has run.

When values are given, the forward sets them on dm and the backward sets them again before it refreshes the transpose, so the
gradient is that of the forward's matrix even if dm was updated or used by another forward in between.  Afterwards dm holds the
values of the forward whose backward ran last, and after a shifted backward the transpose holds A^T + sigma_(L-1) I: every
backward refreshes it before use.  A multiply's backward sets them only when dL/dx is wanted, for the A^T product: the value
gradient depends on the pattern alone.  offd_val without diag_val is refused.

Not differentiated: x0, and a second backward (the Functions are once_differentiable).
"""
import ctypes as C

import torch
from torch.autograd.function import once_differentiable

from .api import _checked_cuda_vectors, bicg_result

RESULT_BYTES = C.sizeof(bicg_result)


def _rows(dm, name, t):
    """t checked as a CUDA float64 tensor of shape (n_loc,) or (k, n_loc): (t as (k, n_loc), k)"""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: need a CUDA float64 tensor, got {type(t).__name__}")
    n = dm.blk.n_loc
    shape = tuple(t.shape) if t.dim() in (1, 2) and t.shape[-1] == n else (n,)
    _checked_cuda_vectors((name, t, shape))
    return t.view(-1, n), (shape[0] if len(shape) == 2 else 1)


def _results(name, t, k, device):
    """an optional k x 24-byte result tensor as k rows (allocated here when None, on the current stream)"""
    if t is None:
        t = torch.empty(k, RESULT_BYTES, dtype=torch.uint8, device=device)
    if not (isinstance(t, torch.Tensor) and t.dtype == torch.uint8 and t.is_contiguous() and t.numel() == k * RESULT_BYTES):
        raise ValueError(f"{name}: need a contiguous uint8 CUDA tensor of {k} x {RESULT_BYTES} bytes")
    return list(t.view(k, RESULT_BYTES))


def _check_values(diag_val, offd_val):
    if offd_val is not None and diag_val is None:
        raise ValueError("offd_val: given without diag_val (set_values takes both, so the forward would not use it)")


def _set_values(dm, diag_val, offd_val, stream):
    if diag_val is not None:
        dm.set_values_async(diag_val.detach(), None if offd_val is None else offd_val.detach(), stream=stream)


def _value_grads(ctx, dm, u, x, alpha, stream):
    """(grad of diag_val, grad of offd_val) where they are wanted: one value_grad_async over every vector"""
    want_d, want_o = ctx.needs_input_grad[ctx.vals_at], ctx.needs_input_grad[ctx.vals_at + 1]
    if not (want_d or want_o):
        return None, None
    gd, go = dm.value_grad_async(u, x, alpha=alpha, stream=stream)
    return (gd if want_d else None), (go if want_o else None)


class SolveFunction(torch.autograd.Function):
    """x = A^-1 b on a DeviceMatrix, differentiable in b and in the values; see solve_autograd."""

    @staticmethod
    def forward(ctx, dm, b, method, diag_val, offd_val, x0, result, adjoint_result):
        _check_values(diag_val, offd_val)
        b2, k = _rows(dm, "b", b)
        if x0 is not None:
            x0_2, _ = _rows(dm, "x0", x0)
            if x0.shape != b.shape:
                raise ValueError(f"x0: shape {tuple(x0.shape)}, expected {tuple(b.shape)}")
        results = _results("result", result, k, b.device)
        ctx.adjoint_results = _results("adjoint_result", adjoint_result, k, b.device)
        stream = torch.cuda.current_stream(b.device)
        _set_values(dm, diag_val, offd_val, stream)
        x = x0_2.clone() if x0 is not None else torch.zeros_like(b2)
        r = b2.clone()
        for j in range(k):
            dm.solve_async(method, x[j], r[j], result=results[j], stream=stream)
        ctx.dm, ctx.method, ctx.k, ctx.vals_at = dm, method, k, 3
        ctx.save_for_backward(x, diag_val, offd_val)
        return x.view(b.shape)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_x):
        dm, method, k = ctx.dm, ctx.method, ctx.k
        x, diag_val, offd_val = ctx.saved_tensors
        stream = torch.cuda.current_stream(grad_x.device)
        _set_values(dm, diag_val, offd_val, stream)
        mt = dm._adjoint()
        mt.transpose_values_async(dm, stream=stream)
        lam = torch.zeros_like(x)
        r = torch.empty_like(x).copy_(grad_x.reshape(x.shape))     # contiguous rows whatever grad_x's strides are
        for j in range(k):
            mt.solve_async(method, lam[j], r[j], result=ctx.adjoint_results[j], stream=stream)
        gd, go = _value_grads(ctx, dm, lam, x, -1.0, stream)
        grad_b = lam.view(grad_x.shape) if ctx.needs_input_grad[1] else None
        return None, grad_b, None, gd, go, None, None, None


class ShiftedSolveFunction(torch.autograd.Function):
    """X_j = (A + sigma_j I)^-1 b on a DeviceMatrix, differentiable in b, sigma and the values; see shifted_solve_autograd."""

    @staticmethod
    def forward(ctx, dm, b, sigma, method, seed, diag_val, offd_val, x0, adjoint_method, result, adjoint_result):
        _check_values(diag_val, offd_val)
        if not isinstance(sigma, torch.Tensor):
            raise TypeError(f"sigma: need a CUDA float64 tensor, got {type(sigma).__name__}")
        if sigma.dim() != 1:
            raise ValueError(f"sigma: need a 1-d tensor, got shape {tuple(sigma.shape)}")
        n, L = dm.blk.n_loc, int(sigma.numel())
        _checked_cuda_vectors(("b", b, (n,)), ("sigma", sigma, (L,)), *((("x0", x0, (L, n)),) if x0 is not None else ()))
        ctx.adjoint_results = _results("adjoint_result", adjoint_result, L, b.device)
        stream = torch.cuda.current_stream(b.device)
        _set_values(dm, diag_val, offd_val, stream)
        x = x0.detach().clone() if x0 is not None else b.new_zeros((L, n))
        r = b.detach().clone()                     # the solve leaves its seed residual here; b stays as it is
        try:
            dm.shifted_solve_async(method, x, r, sigma.detach(), seed, result=result, stream=stream)
        except RuntimeError as e:
            raise RuntimeError(f"shifted_solve_autograd inside a CUDA graph capture needs dm.prepare_shifted_autograd({method!r}, "
                               f"{L}) before the capture") from e
        ctx.dm, ctx.method, ctx.adjoint_method, ctx.vals_at = dm, method, adjoint_method, 5
        ctx.save_for_backward(x, sigma, diag_val, offd_val)
        return x

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_x):
        dm = ctx.dm
        x, sigma, diag_val, offd_val = ctx.saved_tensors
        L = x.shape[0]
        stream = torch.cuda.current_stream(grad_x.device)
        if dm._t is None and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"a backward through shifted_solve_autograd inside a CUDA graph capture needs "
                               f"dm.prepare_shifted_autograd({ctx.method!r}, {L}) before the capture")
        _set_values(dm, diag_val, offd_val, stream)
        mt = dm._adjoint()
        lam = torch.zeros_like(x)
        g = torch.empty_like(x).copy_(grad_x)       # contiguous rows whatever grad_x's strides are
        try:
            for j in range(L):
                mt.transpose_values_async(dm, stream=stream)
                mt.shift_diagonal_async(sigma[j:j + 1], stream=stream)
                mt.solve_async(ctx.adjoint_method, lam[j], g[j], result=ctx.adjoint_results[j], stream=stream)
        except RuntimeError as e:
            raise RuntimeError(f"a backward through shifted_solve_autograd inside a CUDA graph capture needs "
                               f"dm.prepare_shifted_autograd({ctx.method!r}, {L}, adjoint_method={ctx.adjoint_method!r}) "
                               f"before the capture") from e
        grad_b = grad_sigma = None
        if ctx.needs_input_grad[1]:
            grad_b = lam[0].clone()
            for j in range(1, L):
                grad_b += lam[j]
        if ctx.needs_input_grad[2]:
            grad_sigma = dm.dots_async(lam, x, stream=stream).neg_()
        gd, go = _value_grads(ctx, dm, lam, x, -1.0, stream)
        return None, grad_b, grad_sigma, None, None, gd, go, None, None, None, None


class MultiplyFunction(torch.autograd.Function):
    """y_j = (A + sigma_j I) x_j on a DeviceMatrix, differentiable in x, the values and sigma; see multiply_autograd."""

    @staticmethod
    def forward(ctx, dm, x, diag_val, offd_val, sigma):
        _check_values(diag_val, offd_val)
        x2, _ = _rows(dm, "x", x)
        stream = torch.cuda.current_stream(x.device)
        _set_values(dm, diag_val, offd_val, stream)
        y = torch.empty_like(x2)
        s = sigma.detach() if sigma is not None else None
        dm.multiply_async(x2, y, sigma=s, stream=stream)
        ctx.dm, ctx.vals_at = dm, 2
        ctx.save_for_backward(x2, diag_val, offd_val, s)
        return y.view(x.shape)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        dm = ctx.dm
        x, diag_val, offd_val, sigma = ctx.saved_tensors
        stream = torch.cuda.current_stream(grad_y.device)
        g = grad_y.reshape(x.shape).contiguous()
        grad_x = grad_sigma = None
        if ctx.needs_input_grad[1]:
            # only A^T needs the forward's values: the value gradient depends on the pattern alone
            _set_values(dm, diag_val, offd_val, stream)
            mt = dm._adjoint()
            mt.transpose_values_async(dm, stream=stream)
            grad_x = torch.empty_like(x)
            mt.multiply_async(g, grad_x, sigma=sigma, stream=stream)
            grad_x = grad_x.view(grad_y.shape)
        if ctx.needs_input_grad[4]:
            grad_sigma = dm.dots_async(g, x, stream=stream)
        gd, go = _value_grads(ctx, dm, g, x, 1.0, stream)
        return None, grad_x, gd, go, grad_sigma


def solve_autograd(dm, b, method="bicgstab", diag_val=None, offd_val=None, x0=None, result=None, adjoint_result=None):
    """x = A^-1 b on the DeviceMatrix dm, differentiable in b and in diag_val / offd_val.

    b: a CUDA float64 tensor of shape (n_loc,) or (k, n_loc), one solve per row.  diag_val / offd_val: the matrix's values in
    set_values' block order (offd_val where dm has offd entries); when given, the forward first runs dm.set_values_async with
    them, and the backward sets them again.  x0: the initial guess, same shape as b (zero when None; no gradient flows to it).
    result / adjoint_result: optional contiguous uint8 CUDA tensors of k x 24 bytes that receive the bicg_result of every
    forward and backward solve (read them with decode_result on each 24-byte row).  Everything runs on torch's current stream
    with no host synchronisation; the backward solves A^T lambda = dL/dx from lambda = 0 on dm's transpose.  Inside
    torch.cuda.graph, call dm.prepare_autograd(method) first."""
    return SolveFunction.apply(dm, b, method, diag_val, offd_val, x0, result, adjoint_result)


def shifted_solve_autograd(dm, b, sigma, method="shifted_lopbicgstab", seed=0, diag_val=None, offd_val=None, x0=None,
                           adjoint_method="bicgstab", result=None, adjoint_result=None):
    """X_j = (A + sigma_j I)^-1 b for every shift, one shifted_solve_async on the DeviceMatrix dm; returns X of shape
    (sigma_len, n_loc), differentiable in b, sigma and diag_val / offd_val.

    b: a CUDA float64 tensor of shape (n_loc,), which the solve does not change.  sigma: a 1-d CUDA float64 tensor of the
    shifts.  method / seed: as for shifted_solve_async (a key of SHIFTED_SOLVE_EX, and a seed in [0, sigma_len)).  diag_val /
    offd_val: as for solve_autograd.  x0: initial guesses of shape (sigma_len, n_loc) (zero when None; no gradient flows to
    it).  result: an optional 32-byte uint8 CUDA tensor that receives the forward's bicg_shift_result (decode_shift_result);
    adjoint_result: an optional contiguous uint8 CUDA tensor of sigma_len x 24 bytes that receives the bicg_result of every
    adjoint solve.  The backward runs, for each shift in order, transpose_values_async -> shift_diagonal_async(sigma[j:j+1]) ->
    solve_async(adjoint_method) from lambda_j = 0 on dm's transpose, so it costs sigma_len solves with A^T + sigma_j I; a zero
    dL/dX_j costs no iteration.  Everything runs on torch's current stream with no host synchronisation.  Inside
    torch.cuda.graph, call dm.prepare_shifted_autograd(method, sigma_len, adjoint_method) first.  A^T must store a diagonal
    entry in every row."""
    return ShiftedSolveFunction.apply(dm, b, sigma, method, seed, diag_val, offd_val, x0, adjoint_method, result, adjoint_result)


def multiply_autograd(dm, x, diag_val=None, offd_val=None, sigma=None):
    """y_j = (A + sigma_j I) x_j on the DeviceMatrix dm (multiply_async), differentiable in x, in diag_val / offd_val (given as
    for solve_autograd) and in sigma (None: no shift term; else a CUDA float64 tensor of one shift per row of x).  The
    backward forms dL/dx = (A^T + sigma_j I) dL/dy on dm's transpose, dL/da_e = sum_j (dL/dy_j)_i x_j[c] and
    dL/dsigma_j = <dL/dy_j, x_j> (dots_async, over every rank)."""
    return MultiplyFunction.apply(dm, x, diag_val, offd_val, sigma)
