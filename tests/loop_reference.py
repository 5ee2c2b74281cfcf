"""The four loops of the reference's solver.c, restated call for call with the oracle's primitives (O.spmv, O.daxpy, O.dscal,
O.ddot), so that a test can stop them after any iteration and look at every vector and scalar they leave.

reference_state() is the CPU side of the per-iteration GPU tests (tests/test_gpu_loop_state.py, test_gpu_kernels.py).  Its
operation order is oracle/bicg_oracle.c's, which is pinned bit for bit to the compiled reference; tests/test_loop_reference.py
pins this file to the oracle in turn.

exact=True evaluates every SpMV in long double (O.spmv(..., long_double=True)) and every dot product with math.fsum over the
rounded products.  The distance between the two evaluations is the rounding spread of the case itself: how far a correct
implementation that merely sums in a different order may land from the oracle."""
import math

import numpy as np

# arena slot of every vector the loops use (include/bicgstab_b200.h; y of bicgstab and z of the CA / pipelined loops share one)
ARENA = dict(x=0, r=1, rh=2, p=3, s=4, y=5, z=5, w=6, v=7, t=8, b=9, ax=10)
# layout of bicg_debug_get_scalars()
SCALARS = ("rTr", "rTr_old", "rTs", "rTy", "yTy", "rTw", "wTw", "rTz", "dot_r", "dot_zero", "alpha", "beta", "omega")


def _ops(O, n, ptr, col, val, exact):
    if exact:
        A = lambda x: O.spmv(n, ptr, col, val, x, long_double=True)
        dot = lambda x, y: math.fsum(x * y)
    else:
        A = lambda x: O.spmv(n, ptr, col, val, x)
        dot = O.ddot
    return A, dot


def _run(O, method, ptr, col, val, b, ks, krr, nrr, exact, tol, x0=None):
    """Run from x0 (None: zero) until the loop test of solver.c:86 fails for tolerance `tol` and max_iter = max(ks).  Returns
    ({k: state after iteration k, for the k in ks the loop reaches}, the state the loop ends in)."""
    b = np.ascontiguousarray(b, dtype=np.float64)
    n = b.size
    ptr = np.ascontiguousarray(ptr, dtype=np.uint32)
    col = np.ascontiguousarray(col, dtype=np.uint32)
    val = np.ascontiguousarray(val, dtype=np.float64)
    A, dot = _ops(O, n, ptr, col, val, exact)
    ax, sc = O.daxpy, O.dscal
    want = set(ks)
    max_iter = max(ks)
    out = {}
    x = np.zeros(n) if x0 is None else np.array(x0, dtype=np.float64)
    r = b.copy()
    if method == "pipe_bicgstab_rr" and krr <= 0:
        method = "pipe_bicgstab"                                  # the library's reading of krr <= 0 (solve.cu)

    last = {}

    def keep(k, vecs, scal, hist):
        st = {name: v.copy() for name, v in vecs.items()} | scal | {"hist": np.array(hist), "iters": k}
        if k in want:
            out[k] = st
        last["state"] = st                                        # the state the loop ends in, kept whatever k it ends at

    # solver.c:74-79 / 200-203 / 333-336 / 475-479: r = b - A x0, r# = r, (r,r)
    if method == "pipe_bicgstab_rr":
        bb = b.copy()                                             # :475, the caller's b: not r0 unless x0 = 0
    Ax = A(x)
    ax(-1.0, Ax, r)
    rh = r.copy()
    rTr = dot(r, r)
    dot_r = dot_zero = rTr
    hist = [dot_r / dot_zero]
    k = 0
    go = lambda: dot_r > tol * tol * dot_zero and k < max_iter

    if method == "bicgstab":                                      # solver.c:74-120
        p = r.copy()
        while go():
            s = A(p)                                              # :88
            rTs = dot(rh, s)
            alpha = rTr / rTs                                     # :93
            ax(-alpha, s, r)                                      # :94  q, kept in r
            y = A(r)                                              # :96
            rTy, yTy = dot(r, y), dot(y, y)
            omega = rTy / yTy                                     # :104
            ax(alpha, p, x); ax(omega, r, x); ax(-omega, y, r)    # :105-107
            dot_r = dot(r, r)                                     # :108
            rTr_old = rTr
            rTr = dot(rh, r)                                      # :111
            beta = (alpha / omega) * (rTr / rTr_old)              # :116
            k += 1
            hist.append(dot_r / dot_zero)
            # p is the direction this iteration used: the library evaluates the loop test of :86 right after beta, so it never
            # performs the p update of the last pass, whose result the reference computes and then discards (:117-119)
            keep(k, dict(x=x, r=r, rh=rh, p=p, s=s, y=y, ax=Ax),
                 dict(rTr=rTr, rTr_old=rTr_old, rTs=rTs, rTy=rTy, yTy=yTy, dot_r=dot_r, dot_zero=dot_zero,
                      alpha=alpha, beta=beta, omega=omega), hist)
            if not go():
                break
            sc(beta, p); ax(1.0, r, p); ax(-beta * omega, s, p)  # :117-119
        return out, last.get("state")

    # ca_bicgstab solver.c:200-253; pipe_bicgstab :333-388; pipe_bicgstab_rr :433-547.  omega starts at 0 and p, s, z, v, t at
    # zero (DESIGN section 1: the reference reads them uninitialised)
    pipe = method != "ca_bicgstab"
    rr = method == "pipe_bicgstab_rr"
    w = A(r)                                                      # :205 / :338 / :481
    rTw = dot(r, w)
    p, s, z, v, t = (np.zeros(n) for _ in range(5))
    if pipe:
        t = A(w)                                                  # :341 / :484
    alpha, beta, omega = rTr / rTw, 0.0, 0.0
    while go():
        replace = rr and k % krr == 0 and k > 0 and k <= krr * nrr    # :498, :522
        ax(-omega, s, p); sc(beta, p); ax(1.0, r, p)              # :217-219 / :352-354 / :494-496
        if not pipe:
            ax(-omega, z, s); sc(beta, s); ax(1.0, w, s)          # :220-222
            z = A(s)                                              # :224
        elif replace:
            s = A(p)                                              # :499
            z = A(s)                                              # :500
        else:
            ax(-omega, z, s); sc(beta, s); ax(1.0, w, s)          # :355-357
            ax(-omega, v, z); sc(beta, z); ax(1.0, t, z)          # :358-360
        ax(-alpha, s, r)                                          # q
        ax(-alpha, z, w)                                          # y, kept in w
        qy, yy = dot(r, w), dot(w, w)
        if pipe:
            v = A(z)                                              # :365
        omega = qy / yy                                           # :232 / :369
        ax(alpha, p, x); ax(omega, r, x)                          # :233-234 / :370-371
        if replace:
            Ax = A(x)                                             # :523
            r = bb.copy(); ax(-1.0, Ax, r)                        # :524-525
            w = A(r)                                              # :526
        else:
            ax(-omega, w, r)                                      # :235 / :372
            if pipe:
                ax(-alpha, v, t); ax(-omega, t, w)                # :374-375
        dot_r = dot(r, r)                                         # :236 / :373
        if not pipe:
            w = A(r)                                              # :238
        rTr_old = rTr
        rTr, rTw, rTs, rTz = dot(rh, r), dot(rh, w), dot(rh, s), dot(rh, z)
        if pipe:
            t = A(w)                                              # :381
        beta = (alpha / omega) * (rTr / rTr_old)                  # :248 / :387
        alpha = rTr / (rTw + beta * (rTs - omega * rTz))          # :249 / :388
        k += 1
        hist.append(dot_r / dot_zero)
        vecs = dict(x=x, r=r, rh=rh, p=p, s=s, z=z, w=w, ax=Ax)
        if pipe:
            vecs |= dict(v=v, t=t)
        if rr:
            vecs["b"] = bb
        keep(k, vecs, dict(rTr=rTr, rTr_old=rTr_old, rTw=rTw, wTw=yy, rTs=rTs, rTz=rTz, dot_r=dot_r, dot_zero=dot_zero,
                           alpha=alpha, beta=beta, omega=omega), hist)
    return out, last.get("state")


def reference_state(O, method, ptr, col, val, b, k, krr=0, nrr=0, exact=False, tol=0.0, x0=None):
    """Every arena vector the reference leaves defined after iteration k (or after its last iteration, if the loop stops
    earlier on `tol`), with the scalars the library keeps, "hist" (dot_r / dot_zero after iterations 0..k) and "iters".
    x0 is the initial guess (None: zero); exact=True also evaluates its A x0 in long double."""
    return _run(O, method, ptr, col, val, b, [k], krr, nrr, exact, tol, x0)[1]


def reference_states(O, method, ptr, col, val, b, ks, krr=0, nrr=0, exact=False, tol=0.0, x0=None):
    """reference_state() for every k in `ks`, in one pass: {k: state}; a k the loop does not reach is absent.  A state
    holds the vectors under their arena names (ARENA) and the scalars under the names of SCALARS."""
    return _run(O, method, ptr, col, val, b, ks, krr, nrr, exact, tol, x0)[0]
