"""K-level GPU parity (-m gpu): every fused vector phase, every SpMV-epilogue dot and one complete iteration of each
loop, against the reference's own BLAS-1 call sequences (solver.c) executed with the oracle's primitives
(orc_daxpy / orc_dscal / orc_ddot / orc_spmv = vector.c:3-27, matrix.c:498-516) on identical inputs.

Tolerance (SURVEY.md 8(c)): <= 1e-13 relative, max-norm for vectors; dots relative to sum |x_i y_i| (the condition
number of a dot product is not the kernel's business).  Element-wise updates use the same FMA contraction as gcc's
build of the reference, so vectors normally agree bit for bit; only the summation order of the dots differs."""
import ctypes as C

import numpy as np
import pytest

from loop_reference import reference_state

pytestmark = pytest.mark.gpu

V = dict(x=0, r=1, rh=2, p=3, s=4, y=5, z=5, w=6, v=7, t=8, b=9, ax=10)
NV = 11
PH = dict(BICG_INIT=0, BICG_Q=1, BICG_XR=2, BICG_P=3, INIT_R=4, CA_PS=5, QY=6, CA_XR=7, PIPE_1=8, PIPE_3=9,
          RR_P=10, RR_X=11, RR_R=12, RR_DOTS=13)
KTOL = 1e-13


def _ref_phase(O, name, a, al, be, om):
    """The reference's call sequence for the phase (solver.c lines in the comments); a: dict name -> array, in place.
    Returns the list of (x, y) pairs whose dot products the phase reduces, in the kernel's order."""
    ax, sc, dots = O.daxpy, O.dscal, []
    if name in ("BICG_INIT", "INIT_R"):                       # solver.c:75-78 / 201-203
        ax(-1.0, a["ax"], a["r"]); a["rh"][:] = a["r"]
        if name == "BICG_INIT":
            a["p"][:] = a["r"]
        dots = [("r", "r")]
    elif name == "BICG_Q":                                    # :94
        ax(-al, a["s"], a["r"])
    elif name == "BICG_XR":                                   # :105-111
        ax(al, a["p"], a["x"]); ax(om, a["r"], a["x"]); ax(-om, a["y"], a["r"])
        dots = [("r", "r"), ("rh", "r")]
    elif name == "BICG_P":                                    # :117-119
        sc(be, a["p"]); ax(1.0, a["r"], a["p"]); ax(-be * om, a["s"], a["p"])
    elif name == "CA_PS":                                     # :217-222
        ax(-om, a["s"], a["p"]); sc(be, a["p"]); ax(1.0, a["r"], a["p"])
        ax(-om, a["z"], a["s"]); sc(be, a["s"]); ax(1.0, a["w"], a["s"])
    elif name == "QY":                                        # :225-228
        ax(-al, a["s"], a["r"]); ax(-al, a["z"], a["w"])
        dots = [("r", "w"), ("w", "w")]
    elif name == "CA_XR":                                     # :233-236
        ax(al, a["p"], a["x"]); ax(om, a["r"], a["x"]); ax(-om, a["w"], a["r"])
        dots = [("r", "r")]
    elif name == "PIPE_1":                                    # :352-364
        ax(-om, a["s"], a["p"]); sc(be, a["p"]); ax(1.0, a["r"], a["p"])
        ax(-om, a["z"], a["s"]); sc(be, a["s"]); ax(1.0, a["w"], a["s"])
        ax(-om, a["v"], a["z"]); sc(be, a["z"]); ax(1.0, a["t"], a["z"])
        ax(-al, a["s"], a["r"]); ax(-al, a["z"], a["w"])
        dots = [("r", "w"), ("w", "w")]
    elif name == "PIPE_3":                                    # :370-380
        ax(al, a["p"], a["x"]); ax(om, a["r"], a["x"]); ax(-om, a["w"], a["r"])
        ax(-al, a["v"], a["t"]); ax(-om, a["t"], a["w"])
        dots = [("rh", "r"), ("rh", "w"), ("rh", "s"), ("rh", "z"), ("r", "r")]
    elif name == "RR_P":                                      # :494-496
        ax(-om, a["s"], a["p"]); sc(be, a["p"]); ax(1.0, a["r"], a["p"])
    elif name == "RR_X":                                      # :518-519
        ax(al, a["p"], a["x"]); ax(om, a["r"], a["x"])
    elif name == "RR_R":                                      # :524-525
        a["r"][:] = a["b"]; ax(-1.0, a["ax"], a["r"])
    elif name == "RR_DOTS":                                   # :533-539
        dots = [("rh", "r"), ("rh", "w"), ("rh", "s"), ("rh", "z"), ("r", "r")]
    return dots


def _arena(rng, n):
    return np.ascontiguousarray(rng.standard_normal((NV, n)))


def _views(buf):
    return {k: buf[i] for k, i in V.items() if k != "y"} | {"y": buf[V["y"]]}


def _check_dots(O, a, pairs, got):
    for k, (u, v) in enumerate(pairs):
        want = O.ddot(a[u], a[v])
        scale = float(np.abs(a[u] * a[v]).sum()) + 1e-300
        assert abs(got[k] - want) <= KTOL * scale, (k, u, v, got[k], want)


@pytest.mark.parametrize("name", list(PH))
@pytest.mark.parametrize("n", [5003, 262144 + 7])
def test_vec_phase_matches_reference_blas1(B, O, name, n):
    B.set_options(quiet=1, mega=1)
    blk = B.gen_block("laplace5", int(np.ceil(np.sqrt(n))), 0.0)      # any matrix with >= n rows; only the arena is used
    n = blk.n
    dm = B.DeviceMatrix(blk)
    rng = np.random.default_rng(PH[name] * 977 + n)
    buf = _arena(rng, n)
    want = buf.copy()
    al, be, om = 0.7310585786300049, -1.3132616875182228, 0.4189758030700723
    coef = (C.c_double * 3)(al, be, om)
    dots = (C.c_double * 8)()
    nd = B.lib.bicg_debug_vec_phase(dm.h, PH[name], coef, buf.ctypes.data_as(C.c_void_p), dots)
    a = _views(want)
    pairs = _ref_phase(O, name, a, al, be, om)
    assert nd == len(pairs)
    skip = {"t"} if name == "PIPE_3" else set()      # t - alpha v is consumed in registers: t is overwritten by t = A w next
    for k, i in V.items():
        if k in skip:
            continue
        err = np.abs(buf[i] - want[i]).max() / max(np.abs(want[i]).max(), 1e-300)
        assert err <= KTOL, (name, k, err)
    _check_dots(O, a, pairs, list(dots))
    dm.destroy()


@pytest.mark.parametrize("epi", [0, 1, 2, 3])
@pytest.mark.parametrize("kind,g,p0", [("stencil15", 20, 14.0), ("random", 20011, 32)])
def test_spmv_epilogue_dots(B, O, epi, kind, g, p0):
    B.set_options(quiet=1)
    blk = B.gen_block(kind, g, p0)
    n = blk.n
    ptr, col, val = B.block_to_global_csr(blk)
    dm = B.DeviceMatrix(blk)
    buf = _arena(np.random.default_rng(epi + 31 * g), n)
    a = _views(buf.copy())
    dots = (C.c_double * 8)()
    nd = B.lib.bicg_debug_spmv_epi(dm.h, epi, buf.ctypes.data_as(C.c_void_p), dots)
    y = O.spmv(n, ptr, col, val, a["p"])
    out = buf[V["w"]] if epi == 3 else buf[V["s"]]
    assert np.abs(out - y).max() <= KTOL * np.abs(y).max()
    a["Y"] = y
    pairs = {0: [], 1: [("rh", "Y")], 2: [("r", "Y"), ("Y", "Y")],
             3: [("rh", "r"), ("rh", "Y"), ("rh", "ax"), ("rh", "z")]}[epi]
    assert nd == len(pairs)
    _check_dots(O, a, pairs, list(dots))
    dm.destroy()


def _one_iteration_reference(O, method, n, ptr, col, val, b):
    """One pass of the reference loop (tests/loop_reference.py); returns the vectors and scalars it leaves.  p of bicgstab is
    the direction the pass used: the library evaluates the loop test of solver.c:86 right after beta and skips the p update
    whose result the reference computes and then discards."""
    st = reference_state(O, method, ptr, col, val, b, 1)
    names = ("x", "r", "p", "s", "y") if method == "bicgstab" else ("x", "r", "p", "s", "z", "w")
    return {k: st[k] for k in names}, {k: st[k] for k in ("alpha", "omega", "beta", "dot_r")}


@pytest.mark.parametrize("mega", [1, 0], ids=["mega", "multikernel"])
@pytest.mark.parametrize("method", ["bicgstab", "ca_bicgstab"])
@pytest.mark.parametrize("kind,g,p0", [("stencil15", 24, 14.0), ("convdiff", 150, 1.5)])
def test_one_iteration_every_vector_and_scalar(B, O, mega, method, kind, g, p0):
    """Both loop implementations after exactly one iteration: x, r, p, s, y/z, w and alpha, omega, beta, (r,r)."""
    B.set_options(quiet=1, tol=0.0, max_iter=1, mega=mega)
    blk = B.gen_block(kind, g, p0)
    n = blk.n
    ptr, col, val = B.block_to_global_csr(blk)
    dm = B.DeviceMatrix(blk)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    x = np.zeros(n); r = b.copy()
    it, st = dm.solve(method, x, r)
    assert it == 1
    if mega:
        assert st["kernel_launches"] <= 8                       # init kernels + ONE persistent kernel
    vecs, scal = _one_iteration_reference(O, method, n, ptr, col, val, b)
    got = np.empty(n)
    for k, want in vecs.items():
        B.lib.bicg_debug_get_vec(dm.h, V[k], got.ctypes.data_as(C.c_void_p))
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 1e-12, (k, err)           # one SpMV deep: 1e-13 per kernel, a few kernels chained
    s13 = (C.c_double * 13)()
    B.lib.bicg_debug_get_scalars(dm.h, s13)
    gs = dict(dot_r=s13[8], alpha=s13[10], beta=s13[11], omega=s13[12])
    for k, want in scal.items():
        assert abs(gs[k] - want) <= 1e-12 * abs(want), (k, gs[k], want)
    assert np.abs(x - vecs["x"]).max() <= 1e-12 * np.abs(vecs["x"]).max()
    dm.destroy()
    B.set_options(tol=1e-15, max_iter=1000, mega=1)
