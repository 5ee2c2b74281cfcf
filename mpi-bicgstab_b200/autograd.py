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

When values are given, the forward sets them on dm and the backward sets them again, so the gradient is that of the forward's
matrix even if dm was updated or used by another forward in between; the transpose gets them permuted by
DeviceMatrix.transpose_entries_async, which gives the bits transpose_values would.  Without values the transpose is refreshed
from dm: so is the transpose dm keeps for its backward (dm._t) whenever solve_autograd or multiply_autograd runs on it without
values.  Afterwards dm holds the values of the forward whose backward ran last, also after a second backward, and after a
shifted backward the transpose holds A^T + sigma_(L-1) I: every backward sets it before use.  A multiply's backward sets them only when dL/dx is wanted, for the
A^T product: the value gradient depends on the pattern alone.  offd_val without diag_val is refused.

Every backward is itself a composition of differentiable Functions, so torch.autograd.grad(..., create_graph=True) and
torch.autograd.functional.hvp work to any order: the adjoint solve is a SolveFunction on the transpose (whose adjoint is dm
again: the transpose made for a backward links back to its source), and the value gradient, the weighted multiply
(DeviceMatrix.multiply_values_async, the derivative of the value gradient), the entry permutation between dm and its
transpose, and the dot products each have a Function whose backward uses the others.  A first-order backward
(create_graph=False) runs the same kernels on the same data as before this was so, and gives the same bits.  A second backward
inside torch.cuda.graph needs the same prepare_autograd / prepare_shifted_autograd as the first.  A second backward through a
shifted solve needs its values as diag_val / offd_val (constants will do): its adjoint solves shift A itself by sigma_j, and a
shift accumulates on the stored values, so they are set before each shift and again afterwards; without them it raises.

Not differentiated: x0 (the gradient in it is zero at convergence).
"""
import ctypes as C

import torch

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


def _value_grads(ctx, dm, u, x, alpha):
    """(grad of diag_val, grad of offd_val) where they are wanted: one value gradient over every vector"""
    want_d, want_o = ctx.needs_input_grad[ctx.vals_at], ctx.needs_input_grad[ctx.vals_at + 1]
    if not (want_d or want_o):
        return None, None
    gd, go = _ValueGrad.apply(dm, u, x, alpha)
    return (gd if want_d else None), (go if want_o else None)


def _refresh_or_set(dm, diag_val, offd_val, stream):
    """the forward's values on dm: the given ones, else, on a transpose made for a backward, its source's current values"""
    if diag_val is not None:
        _set_values(dm, diag_val, offd_val, stream)
    elif dm._src is not None:
        dm.transpose_values_async(dm._src, stream=stream)


def _permute(dm, pair, wd, wo):
    """an entry vector of dm in the block order of pair = dm._adjoint(), differentiably (None when wd is None)"""
    if wd is None:
        return None, None
    if dm._src is not None:                       # dm is the transpose and pair its source
        return _TransposeEntries.apply(dm, pair, True, wd, wo)
    return _TransposeEntries.apply(pair, dm, False, wd, wo)


class _TransposeEntries(torch.autograd.Function):
    """(out_diag, out_offd) = mt.transpose_entries_async(src, in, reverse); the adjoint of a permutation is its inverse."""

    @staticmethod
    def forward(ctx, mt, src, reverse, in_diag, in_offd):
        ctx.mt, ctx.src, ctx.reverse = mt, src, reverse
        return mt.transpose_entries_async(src, in_diag.detach(), None if in_offd is None else in_offd.detach(), reverse=reverse,
                                          stream=torch.cuda.current_stream(in_diag.device))

    @staticmethod
    def backward(ctx, g_diag, g_offd):
        gd, go = _TransposeEntries.apply(ctx.mt, ctx.src, not ctx.reverse, g_diag.contiguous(),
                                         None if g_offd is None else g_offd.contiguous())
        return None, None, None, gd, (go if ctx.needs_input_grad[4] else None)


class _ValueGrad(torch.autograd.Function):
    """(g_diag, g_offd) = dm.value_grad_async(u, v, alpha): g_e = alpha sum_j u_j[i] v_j[c] over the pattern.  With weights
    W = dL/dg: dL/du = alpha A_W v, dL/dv = alpha A_W^T u (the weighted multiply on the transpose, W permuted there)."""

    @staticmethod
    def forward(ctx, dm, u, v, alpha):
        ctx.dm, ctx.alpha = dm, alpha
        ctx.save_for_backward(u, v)
        return dm.value_grad_async(u.detach(), v.detach(), alpha=alpha, stream=torch.cuda.current_stream(u.device))

    @staticmethod
    def backward(ctx, w_diag, w_offd):
        dm, alpha = ctx.dm, ctx.alpha
        u, v = ctx.saved_tensors
        w_diag = w_diag.contiguous()
        w_offd = None if w_offd is None else w_offd.contiguous()
        gu = gv = None
        if ctx.needs_input_grad[1]:
            gu = _MultiplyValues.apply(dm, w_diag, w_offd, v, alpha)
        if ctx.needs_input_grad[2]:
            pair = dm._adjoint()
            pd, po = _permute(dm, pair, w_diag, w_offd)
            gv = _MultiplyValues.apply(pair, pd, po, u, alpha)
        return None, gu, gv, None


class _MultiplyValues(torch.autograd.Function):
    """y = alpha A_W x on dm's pattern with weights W (dm.multiply_values_async).  dL/dW = the value gradient of (dL/dy, x)
    with alpha; dL/dx = alpha A_W^T dL/dy on the transpose."""

    @staticmethod
    def forward(ctx, dm, w_diag, w_offd, x, alpha):
        ctx.dm, ctx.alpha = dm, alpha
        ctx.save_for_backward(w_diag, w_offd, x)
        return dm.multiply_values_async(w_diag.detach(), None if w_offd is None else w_offd.detach(), x.detach(), alpha=alpha,
                                        stream=torch.cuda.current_stream(x.device))

    @staticmethod
    def backward(ctx, grad_y):
        dm, alpha = ctx.dm, ctx.alpha
        w_diag, w_offd, x = ctx.saved_tensors
        g = grad_y.contiguous()
        gd = go = gx = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            gd, go = _ValueGrad.apply(dm, g, x, alpha)
        if ctx.needs_input_grad[3]:
            pair = dm._adjoint()
            pd, po = _permute(dm, pair, w_diag, w_offd)
            gx = _MultiplyValues.apply(pair, pd, po, g, alpha)
        return (None, gd if ctx.needs_input_grad[1] else None, go if ctx.needs_input_grad[2] else None, gx, None)


class _Dots(torch.autograd.Function):
    """out_j = <u_j, v_j> over every rank (dm.dots_async).  dL/du_j = dL/dout_j v_j, dL/dv_j = dL/dout_j u_j: rank-local, since
    every rank holds the same dL/dout."""

    @staticmethod
    def forward(ctx, dm, u, v):
        ctx.save_for_backward(u, v)
        return dm.dots_async(u.detach(), v.detach(), stream=torch.cuda.current_stream(u.device))

    @staticmethod
    def backward(ctx, grad_out):
        u, v = ctx.saved_tensors
        o = grad_out.unsqueeze(-1) if u.dim() == 2 else grad_out
        return (None, o * v if ctx.needs_input_grad[1] else None, o * u if ctx.needs_input_grad[2] else None)


class SolveFunction(torch.autograd.Function):
    """x = (A + sigma I)^-1 b on a DeviceMatrix, differentiable in b, in the values and in sigma; see solve_autograd.  sigma
    (internal: one device value, or None) is what the adjoint solves of a shifted backward use."""

    @staticmethod
    def forward(ctx, dm, b, method, diag_val, offd_val, x0, result, adjoint_result, sigma=None):
        _check_values(diag_val, offd_val)
        b2, k = _rows(dm, "b", b)
        if x0 is not None:
            x0_2, _ = _rows(dm, "x0", x0)
            if x0.shape != b.shape:
                raise ValueError(f"x0: shape {tuple(x0.shape)}, expected {tuple(b.shape)}")
        results = _results("result", result, k, b.device)
        ctx.adjoint_result = adjoint_result
        if adjoint_result is not None:
            _results("adjoint_result", adjoint_result, k, b.device)    # checked here, filled by the backward's solve
        # a shift accumulates on the stored values: a handle that is not a transpose made for a backward cannot refresh them, so
        # it shifts only values given here, and holds them again afterwards
        own = sigma is not None and dm._src is None
        if own and diag_val is None:
            raise RuntimeError("a second derivative through shifted_solve_autograd needs the matrix's values as diag_val / "
                               "offd_val (they may be constants): its adjoint solves on A + sigma_j I set them before each shift")
        stream = torch.cuda.current_stream(b.device)
        _refresh_or_set(dm, diag_val, offd_val, stream)
        if sigma is not None:
            dm.shift_diagonal_async(sigma.detach(), stream=stream)
        x = x0_2.clone() if x0 is not None else torch.zeros_like(b2)
        r = b2.detach().clone()
        for j in range(k):
            dm.solve_async(method, x[j], r[j], result=results[j], stream=stream)
        if own:
            _set_values(dm, diag_val, offd_val, stream)
        out = x.view(b.shape)
        ctx.dm, ctx.method, ctx.vals_at = dm, method, 3
        ctx.save_for_backward(out, diag_val, offd_val, sigma)
        return out

    @staticmethod
    def backward(ctx, grad_x):
        dm = ctx.dm
        out, diag_val, offd_val, sigma = ctx.saved_tensors
        x = out.reshape(-1, dm.blk.n_loc)
        stream = torch.cuda.current_stream(grad_x.device)
        _set_values(dm, diag_val, offd_val, stream)
        pair = dm._adjoint()
        pd, po = _permute(dm, pair, diag_val, offd_val)
        g = grad_x.reshape(x.shape).contiguous()
        lam = SolveFunction.apply(pair, g, ctx.method, pd, po, None, ctx.adjoint_result, None, sigma)
        grad_b = lam.reshape(grad_x.shape) if ctx.needs_input_grad[1] else None
        grad_sigma = None
        if sigma is not None and ctx.needs_input_grad[8]:
            grad_sigma = -_Dots.apply(dm, lam, x).sum().reshape(sigma.shape)
        gd, go = _value_grads(ctx, dm, lam, x, -1.0)
        return None, grad_b, None, gd, go, None, None, None, grad_sigma


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
        pd, po = _permute(dm, mt, diag_val, offd_val)
        g = grad_x.contiguous()
        try:
            lam = torch.stack([SolveFunction.apply(mt, g[j], ctx.adjoint_method, pd, po, None, ctx.adjoint_results[j], None,
                                                   sigma[j:j + 1]) for j in range(L)])
        except RuntimeError as e:
            raise RuntimeError(f"a backward through shifted_solve_autograd inside a CUDA graph capture needs "
                               f"dm.prepare_shifted_autograd({ctx.method!r}, {L}, adjoint_method={ctx.adjoint_method!r}) "
                               f"before the capture") from e
        grad_b = grad_sigma = None
        if ctx.needs_input_grad[1]:
            grad_b = lam[0]
            for j in range(1, L):
                grad_b = grad_b + lam[j]
        if ctx.needs_input_grad[2]:
            grad_sigma = -_Dots.apply(dm, lam, x)
        gd, go = _value_grads(ctx, dm, lam, x, -1.0)
        return None, grad_b, grad_sigma, None, None, gd, go, None, None, None, None


class MultiplyFunction(torch.autograd.Function):
    """y_j = (A + sigma_j I) x_j on a DeviceMatrix, differentiable in x, the values and sigma; see multiply_autograd."""

    @staticmethod
    def forward(ctx, dm, x, diag_val, offd_val, sigma):
        _check_values(diag_val, offd_val)
        x2, _ = _rows(dm, "x", x)
        stream = torch.cuda.current_stream(x.device)
        _refresh_or_set(dm, diag_val, offd_val, stream)
        y = torch.empty_like(x2)
        dm.multiply_async(x2.detach(), y, sigma=sigma.detach() if sigma is not None else None, stream=stream)
        ctx.dm, ctx.vals_at = dm, 2
        ctx.save_for_backward(x, diag_val, offd_val, sigma)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, grad_y):
        dm = ctx.dm
        x, diag_val, offd_val, sigma = ctx.saved_tensors
        x2 = x.reshape(-1, dm.blk.n_loc)
        stream = torch.cuda.current_stream(grad_y.device)
        g = grad_y.reshape(x2.shape).contiguous()
        grad_x = grad_sigma = None
        if ctx.needs_input_grad[1]:
            # only A^T needs the forward's values: the value gradient depends on the pattern alone
            _set_values(dm, diag_val, offd_val, stream)
            pair = dm._adjoint()
            pd, po = _permute(dm, pair, diag_val, offd_val)
            grad_x = MultiplyFunction.apply(pair, g, pd, po, sigma).reshape(grad_y.shape)
        if ctx.needs_input_grad[4]:
            grad_sigma = _Dots.apply(dm, g, x2)
        gd, go = _value_grads(ctx, dm, g, x2, 1.0)
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
    entry in every row.  A second derivative (create_graph=True, then a second backward) needs diag_val / offd_val, which may
    be constants: its solves with A + sigma_j I shift A itself and set the values before and after; without them it raises."""
    return ShiftedSolveFunction.apply(dm, b, sigma, method, seed, diag_val, offd_val, x0, adjoint_method, result, adjoint_result)


def multiply_autograd(dm, x, diag_val=None, offd_val=None, sigma=None):
    """y_j = (A + sigma_j I) x_j on the DeviceMatrix dm (multiply_async), differentiable in x, in diag_val / offd_val (given as
    for solve_autograd) and in sigma (None: no shift term; else a CUDA float64 tensor of one shift per row of x).  The
    backward forms dL/dx = (A^T + sigma_j I) dL/dy on dm's transpose, dL/da_e = sum_j (dL/dy_j)_i x_j[c] and
    dL/dsigma_j = <dL/dy_j, x_j> (dots_async, over every rank)."""
    return MultiplyFunction.apply(dm, x, diag_val, offd_val, sigma)
