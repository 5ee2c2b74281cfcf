"""GPU: second derivatives through solves and products on a resident matrix, and the two device operations the differentiable
backward is built from: the multiply with caller weights on a handle's pattern (multiply_values_async) and the permutation of
entry vectors between a handle and its transpose (transpose_entries_async).
Checked: both operations bit for bit (the weighted multiply against multiply_async on both SpMV plan kinds, the permutation
against transpose_values and as an exact round trip); Hessian-vector products and double backward of solve_autograd,
multiply_autograd and shifted_solve_autograd against dense torch.linalg.solve; gradgradcheck; first-order gradients
unchanged by a double backward; an HVP captured in torch.cuda.graph and replayed."""
import numpy as np
import pytest

from test_gpu_autograd import _bits, _cuda, _perturbed, small_csr
from test_gpu_transpose import _case_csr

pytestmark = pytest.mark.gpu

SIGMA = np.array([0.0, 0.5, 1.25])


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, tol=1e-14, max_iter=3000, shift_tol=1e-14, shift_max_iter=3000, mega=1, resident=1,
                  spmv="auto")
    yield
    B.set_options(tol=1e-15, max_iter=1000, shift_tol=1e-12, shift_max_iter=1000, mega=1, resident=1, spmv="auto")


def _torch():
    import torch
    return torch


def _csr(B, case):
    if case == "tprime64":
        blk = B.gen_block("stencil15", 64, 14.0)
        ptr, col, val = (np.asarray(a) for a in B.block_to_global_csr(blk))
        val = val * (1.0 + (np.repeat(np.arange(blk.n), np.diff(ptr)) % 5) / 16.0)
        return blk.n, ptr.astype(np.int64), col.astype(np.int64), val.astype(np.float64)
    return small_csr(B, case)


def _handle(B, n, ptr, col, val):
    return B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))


# ---- the weighted multiply --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spmv", ["tma", "rowsplit"])
@pytest.mark.parametrize("case", ["convdiff", "golden", "tprime8", "tprime64"])
def test_multiply_values_bits(B, case, spmv):
    """W = the handle's own values: multiply_values_async equals multiply_async bit for bit for nvec 1, 3, 8, 9 and several
    alpha / beta (beta = 0 with y full of NaN); W read from a misaligned view, and other weights against set_values + multiply"""
    torch = _torch()
    B.set_options(spmv=spmv)
    n, ptr, col, val = _csr(B, case)
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(3)
        w = _cuda(_perturbed(val, 1))
        dm.set_values_async(w)
        for nvec in (1, 3, 8, 9):
            x = _cuda(rng.standard_normal((nvec, n)))
            y0 = rng.standard_normal((nvec, n))
            for alpha, beta in ((1.0, 0.0), (1.5, 0.0), (-0.75, 1.0), (2.0, -0.5)):
                init = np.full((nvec, n), np.nan) if beta == 0.0 else y0
                want, got = _cuda(init), _cuda(init)
                dm.multiply_async(x, want, alpha=alpha, beta=beta)
                dm.multiply_values_async(w, None, x, got, alpha=alpha, beta=beta)
                torch.cuda.synchronize()
                assert not torch.isnan(got).any()
                assert _bits(got) == _bits(want), (case, spmv, nvec, alpha, beta)
        x = _cuda(rng.standard_normal((3, n)))
        buf = torch.zeros(w.numel() + 1, dtype=torch.float64, device="cuda")
        buf[1:] = w
        want = dm.multiply_values_async(w, None, x)
        got = dm.multiply_values_async(buf[1:], None, x)                 # 8-byte aligned only: staged
        w2 = _cuda(_perturbed(val, 2))
        got2 = dm.multiply_values_async(w2, None, x)
        dm.set_values_async(w2)
        want2 = torch.empty_like(x)
        dm.multiply_async(x, want2)
        torch.cuda.synchronize()
        assert _bits(got) == _bits(want) and _bits(got2) == _bits(want2)
    finally:
        dm.destroy()


# ---- the entry permutation --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["convdiff", "random", "tprime", "golden", "handmade"])
def test_transpose_entries_bits(B, case):
    """forward(values) then set_values on the transpose gives the spmv and solve bits of transpose_values; reverse(forward(r))
    and forward(reverse(s)) give back r and s bit for bit on random vectors (duplicates and explicit zeros included)"""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, case)
    dm = _handle(B, n, ptr, col, val)
    mt = dm._adjoint()
    try:
        rng = np.random.default_rng(5)
        vals = _cuda(_perturbed(val, 3))
        dm.set_values_async(vals)
        mt.transpose_values_async(dm)
        x = rng.standard_normal(n)
        B.set_options(tol=1e-10)

        def state():
            xs, rs = np.zeros(n), x.copy()
            it, _ = mt.solve("bicgstab", xs, rs)
            return _bits(mt.spmv(x)), it, _bits(xs), _bits(rs)
        want = state()
        pd, po = mt.transpose_entries_async(dm, vals)
        mt.set_values_async(pd, po)
        torch.cuda.synchronize()
        assert state() == want
        r = _cuda(rng.standard_normal(val.size))
        r[::7] = 0.0
        fd, fo = mt.transpose_entries_async(dm, r)
        back, _ = mt.transpose_entries_async(dm, fd, fo, reverse=True)
        s = _cuda(rng.standard_normal(int(mt.blk.diag.nz)))
        sd, _ = mt.transpose_entries_async(dm, s, reverse=True)
        s2, _ = mt.transpose_entries_async(dm, sd)
        torch.cuda.synchronize()
        assert _bits(back) == _bits(r) and _bits(s2) == _bits(s)
        assert sorted(_bits(fd)[i:i + 8] for i in range(0, 8 * val.size, 8)) == \
            sorted(_bits(r)[i:i + 8] for i in range(0, 8 * val.size, 8))
    finally:
        dm.destroy()
    assert mt.h is None and dm.h is None


def test_back_link(B):
    """the transpose made for a backward has its source as adjoint; destroying it leaves the source working"""
    n, ptr, col, val = _case_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    try:
        mt = dm._adjoint()
        assert mt._adjoint() is dm and mt._t is None
        mt.destroy()
        dm._t = None
        assert dm.h is not None
        x = np.ones(n)
        assert np.isfinite(dm.spmv(x)).all()
    finally:
        dm.destroy()


# ---- second derivatives against dense torch ----------------------------------------------------------------------------
def _dense(torch, n, ptr, col, vals):
    rows = torch.from_numpy(np.repeat(np.arange(n), np.diff(ptr))).cuda()
    cols = torch.from_numpy(np.asarray(col)).cuda()
    return torch.zeros((n, n), dtype=torch.float64, device="cuda").index_put((rows, cols), vals, accumulate=True)


def _loss(torch, x, w):
    return (w * x).sum() + 0.5 * (x * x).sum() + (x[..., :3] ** 3).sum() / 3.0


def _rel(got, want):
    return max(float((g - h).abs().max() / h.abs().max().clamp_min(1e-300)) for g, h in zip(got, want))


def _hvp_and_double(torch, f, inputs, vs):
    """(hvp, grads of <grad f, v> by create_graph=True then a second grad)"""
    _, hv = torch.autograd.functional.hvp(f, inputs, vs)
    ins = [t.detach().clone().requires_grad_(True) for t in inputs]
    g = torch.autograd.grad(f(*ins), ins, create_graph=True)
    gg = torch.autograd.grad(sum((a * v).sum() for a, v in zip(g, vs)), ins)
    return list(hv) + list(gg)


@pytest.mark.parametrize("case", ["convdiff", "golden", "tprime8"])
def test_solve_hvp_against_dense(B, case):
    torch = _torch()
    n, ptr, col, val = small_csr(B, case)
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(11)
        b, vals, w = _cuda(rng.standard_normal(n)), _cuda(_perturbed(val, 1)), _cuda(rng.standard_normal(n))
        vs = (_cuda(rng.standard_normal(n)), _cuda(rng.standard_normal(val.size)))
        got = _hvp_and_double(torch, lambda bb, vv: _loss(torch, B.solve_autograd(dm, bb, diag_val=vv), w), (b, vals), vs)
        want = _hvp_and_double(torch, lambda bb, vv: _loss(torch, torch.linalg.solve(_dense(torch, n, ptr, col, vv), bb), w),
                               (b, vals), vs)
        rel = _rel(got, want)
        print(f"solve hvp {case}: relative deviation {rel:.2e}")
        assert rel <= 1e-8, (case, rel)
    finally:
        dm.destroy()


@pytest.mark.parametrize("case", ["convdiff", "golden", "tprime8"])
def test_multiply_hvp_against_dense(B, case):
    torch = _torch()
    n, ptr, col, val = small_csr(B, case)
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(12)
        x, vals, s = _cuda(rng.standard_normal((3, n))), _cuda(_perturbed(val, 2)), _cuda(SIGMA)
        w = _cuda(rng.standard_normal((3, n)))
        vs = (_cuda(rng.standard_normal((3, n))), _cuda(rng.standard_normal(val.size)), _cuda(rng.standard_normal(3)))
        got = _hvp_and_double(torch, lambda xx, vv, ss: _loss(torch, B.multiply_autograd(dm, xx, diag_val=vv, sigma=ss), w),
                              (x, vals, s), vs)
        want = _hvp_and_double(torch, lambda xx, vv, ss: _loss(torch, xx @ _dense(torch, n, ptr, col, vv).T + ss[:, None] * xx, w),
                               (x, vals, s), vs)
        rel = _rel(got, want)
        print(f"multiply hvp {case}: relative deviation {rel:.2e}")
        assert rel <= 1e-8, (case, rel)
    finally:
        dm.destroy()


@pytest.mark.parametrize("method", ["shifted_lopbicgstab", "shifted_lopbicg_switching"])
@pytest.mark.parametrize("case", ["convdiff", "tprime8"])
def test_shifted_hvp_against_dense(B, case, method):
    torch = _torch()
    n, ptr, col, val = small_csr(B, case)
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(13)
        b, s, vals = _cuda(rng.standard_normal(n)), _cuda(SIGMA), _cuda(_perturbed(val, 1))
        w = _cuda(rng.standard_normal((SIGMA.size, n)))
        vs = (_cuda(rng.standard_normal(n)), _cuda(rng.standard_normal(SIGMA.size)), _cuda(rng.standard_normal(val.size)))
        eye = torch.eye(n, dtype=torch.float64, device="cuda")

        def dense(bb, ss, vv):
            A = _dense(torch, n, ptr, col, vv)
            return torch.stack([torch.linalg.solve(A + ss[j] * eye, bb) for j in range(SIGMA.size)])
        got = _hvp_and_double(torch, lambda bb, ss, vv: _loss(torch, B.shifted_solve_autograd(dm, bb, ss, method, diag_val=vv), w),
                              (b, s, vals), vs)
        want = _hvp_and_double(torch, lambda bb, ss, vv: _loss(torch, dense(bb, ss, vv), w), (b, s, vals), vs)
        rel = _rel(got, want)
        print(f"shifted hvp {case} {method}: relative deviation {rel:.2e}")
        assert rel <= 1e-8, (case, method, rel)
    finally:
        dm.destroy()


@pytest.mark.parametrize("case", ["convdiff", "tprime8"])
def test_shifted_hvp_with_constant_values_keeps_the_matrix(B, case):
    """an HVP in (b, sigma) of a shifted solve whose values are constants agrees with dense torch, and leaves dm's values as
    they were (the adjoint solves on A + sigma_j I set them before each shift and again afterwards): spmv and a later HVP
    give the same bits as before.  Without values, the second backward raises before it shifts anything."""
    torch = _torch()
    n, ptr, col, val = small_csr(B, case)
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(16)
        b, s = _cuda(rng.standard_normal(n)), _cuda(SIGMA)
        vals = _cuda(val)                                       # the handle's own values, no gradient wanted in them
        w = _cuda(rng.standard_normal((SIGMA.size, n)))
        vs = (_cuda(rng.standard_normal(n)), _cuda(rng.standard_normal(SIGMA.size)))
        eye = torch.eye(n, dtype=torch.float64, device="cuda")
        x0 = rng.standard_normal(n)
        spmv0 = _bits(dm.spmv(x0))

        def dense(bb, ss):
            A = _dense(torch, n, ptr, col, vals)
            return torch.stack([torch.linalg.solve(A + ss[j] * eye, bb) for j in range(SIGMA.size)])
        f = lambda bb, ss: _loss(torch, B.shifted_solve_autograd(dm, bb, ss, diag_val=vals), w)      # noqa: E731
        got = _hvp_and_double(torch, f, (b, s), vs)
        torch.cuda.synchronize()
        assert _bits(dm.spmv(x0)) == spmv0
        want = _hvp_and_double(torch, lambda bb, ss: _loss(torch, dense(bb, ss), w), (b, s), vs)
        rel = _rel(got, want)
        print(f"shifted hvp, constant values, {case}: relative deviation {rel:.2e}")
        assert rel <= 1e-8, (case, rel)
        again = _hvp_and_double(torch, f, (b, s), vs)
        assert [_bits(a) for a in again] == [_bits(a) for a in got]
        tb, ts = b.clone().requires_grad_(True), s.clone().requires_grad_(True)
        g = torch.autograd.grad(_loss(torch, B.shifted_solve_autograd(dm, tb, ts), w), (tb, ts), create_graph=True)
        with pytest.raises(RuntimeError, match="needs the matrix's values"):
            torch.autograd.grad((g[0] * vs[0]).sum() + (g[1] * vs[1]).sum(), (tb, ts))
        torch.cuda.synchronize()
        assert _bits(dm.spmv(x0)) == spmv0
    finally:
        dm.destroy()


def test_entry_points_refuse_bad_arguments(B):
    """on a real handle and its transpose: every -1 case of transpose_entries_async (reverse outside {0, 1}, null pointers, an
    output overlapping an input, a handle that is not the other's transpose); after the prepare, a captured
    multiply_values_async on the tile plan takes an 8-byte aligned W"""
    torch = _torch()
    B.set_options(spmv="tma")
    n, ptr, col, val = _case_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    other = _handle(B, n, ptr, col, val)
    try:
        mt = dm._adjoint()
        f = B.lib.bicg_matrix_transpose_entries_async
        r = _cuda(val)
        o = torch.empty_like(r)
        big = torch.zeros(2 * val.size, dtype=torch.float64, device="cuda")
        ip, op_, bp = r.data_ptr(), o.data_ptr(), big.data_ptr()
        st = torch.cuda.current_stream().cuda_stream
        assert f(mt.h, dm.h, 0, ip, None, op_, None, st) == 0 and f(mt.h, dm.h, 1, op_, None, ip, None, st) == 0
        for args in ((mt.h, dm.h, 2, ip, op_), (mt.h, dm.h, -1, ip, op_), (mt.h, dm.h, 0, None, op_), (mt.h, dm.h, 0, ip, None),
                     (mt.h, dm.h, 0, ip, ip), (mt.h, dm.h, 1, bp, bp + 8 * (val.size - 1)), (dm.h, mt.h, 0, ip, op_),
                     (mt.h, other.h, 0, ip, op_), (None, dm.h, 0, ip, op_), (mt.h, None, 0, ip, op_)):
            assert f(args[0], args[1], args[2], args[3], None, args[4], None, st) == -1, args
        with pytest.raises(ValueError, match="-1"):
            mt.transpose_entries_async(other, r)
        dm.prepare_multiply_values_async()
        x = _cuda(np.random.default_rng(2).standard_normal((2, n)))
        y, want = torch.empty_like(x), torch.empty_like(x)
        big[1:1 + val.size] = r
        dm.set_values_async(r)
        dm.multiply_async(x, want)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            dm.multiply_values_async(big[1:1 + val.size], None, x, y)
        g.replay()
        torch.cuda.synchronize()
        assert _bits(y) == _bits(want)
        del g
    finally:
        dm.destroy()
        other.destroy()


def test_gradgradcheck(B):
    """torch.autograd.gradgradcheck on the solve, the multiply and the shifted solve, convdiff g = 8 (n = 64)"""
    torch = _torch()
    blk = B.gen_block("convdiff", 8, 2.0)
    n = blk.n
    dm = B.DeviceMatrix(blk)
    try:
        vals = _cuda(blk.diag_arrays()[0].copy(), True)
        rng = np.random.default_rng(1)
        b, x, s = _cuda(rng.standard_normal(n), True), _cuda(rng.standard_normal((2, n)), True), _cuda(SIGMA[1:], True)
        kw = dict(fast_mode=True, atol=1e-6, rtol=1e-4)
        assert torch.autograd.gradgradcheck(lambda bb, vv: B.solve_autograd(dm, bb, diag_val=vv), (b, vals), **kw)
        assert torch.autograd.gradgradcheck(lambda xx, vv, ss: B.multiply_autograd(dm, xx, diag_val=vv, sigma=ss), (x, vals, s), **kw)
        assert torch.autograd.gradgradcheck(lambda bb, ss, vv: B.shifted_solve_autograd(dm, bb, ss, diag_val=vv), (b, s, vals), **kw)
    finally:
        dm.destroy()


def test_first_order_unchanged_by_double_backward(B):
    """first-order gradients of solve, multiply and shifted solve before and after a double backward on the same handles"""
    torch = _torch()
    n, ptr, col, val = small_csr(B, "convdiff")
    dm = _handle(B, n, ptr, col, val)
    try:
        rng = np.random.default_rng(14)
        b, w, v0 = rng.standard_normal(n), _cuda(rng.standard_normal(n)), _perturbed(val, 1)

        def first():
            tb, tv, ts = _cuda(b, True), _cuda(v0, True), _cuda(SIGMA, True)
            loss = (B.solve_autograd(dm, tb, diag_val=tv) * w).sum() + (B.multiply_autograd(dm, tb, diag_val=tv) * w).sum()
            loss = loss + (B.shifted_solve_autograd(dm, tb, ts, diag_val=tv) * w).sum()
            loss.backward()
            return [_bits(t.grad) for t in (tb, tv, ts)]
        before = first()
        vb, vv = _cuda(rng.standard_normal(n)), _cuda(rng.standard_normal(val.size))
        _hvp_and_double(torch, lambda bb, vals: _loss(torch, B.solve_autograd(dm, bb, diag_val=vals), w), (_cuda(b), _cuda(v0)),
                        (vb, vv))
        assert first() == before
    finally:
        dm.destroy()


def test_graph_capture_hvp(B):
    """after prepare_autograd / prepare_shifted_autograd, an HVP (forward, grad with create_graph, second grad) captured in
    torch.cuda.graph and replayed with a new b equals the eager HVP bit for bit"""
    torch = _torch()
    n, ptr, col, val = small_csr(B, "convdiff")
    rng = np.random.default_rng(15)
    w, vals = _cuda(rng.standard_normal((SIGMA.size, n))), _cuda(_perturbed(val, 1))
    vb, vv = _cuda(rng.standard_normal(n)), _cuda(rng.standard_normal(val.size))
    for shifted in (False, True):
        dm = _handle(B, n, ptr, col, val)
        try:
            if shifted:
                ts = _cuda(SIGMA)
                dm.prepare_shifted_autograd("shifted_lopbicgstab", SIGMA.size)
                fwd = lambda bb, v_: B.shifted_solve_autograd(dm, bb, ts, diag_val=v_)           # noqa: E731
            else:
                dm.prepare_autograd("bicgstab")
                fwd = lambda bb, v_: B.solve_autograd(dm, bb, diag_val=v_)                       # noqa: E731

            def hvp(tb, tv):
                g = torch.autograd.grad(_loss(torch, fwd(tb, tv), w[:1] if not shifted else w), (tb, tv), create_graph=True)
                return torch.autograd.grad((g[0] * vb).sum() + (g[1] * vv).sum(), (tb, tv))
            tb, tv = _cuda(rng.standard_normal(n), True), vals.clone().requires_grad_(True)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                hvp(tb, tv)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = hvp(tb, tv)
            for k in range(2):
                bnew = rng.standard_normal(n)
                with torch.no_grad():
                    tb.copy_(torch.from_numpy(bnew))
                g.replay()
                torch.cuda.synchronize()
                want = hvp(_cuda(bnew, True), vals.clone().requires_grad_(True))
                torch.cuda.synchronize()
                assert [_bits(a) for a in out] == [_bits(a) for a in want], (shifted, k)
            del g
        finally:
            dm.destroy()
