"""The four shifted solvers, restated call for call with the oracle's primitives (O.spmv, O.daxpy, O.dscal, O.ddot), so that a
test can stop them after any iteration and look at every x_j, p_j and per-shift scalar they leave:

  shifted_lopbicg_switching  oracle/bicg_oracle.c orc_shifted_lopbicg_switching (seed switch included)
  shifted_lopbicg            oracle/shifted_fixed_oracle.c orc_shifted_lopbicg
  shifted_lopbicgstab        oracle/shifted_lop_oracle.c orc_shifted_lop, pipe = 0
  shifted_pipe_lopbicgstab   oracle/shifted_lop_oracle.c orc_shifted_lop, pipe = 1

This is the counterpart of tests/loop_reference.py for the shifted solvers: the CPU side of tests/test_gpu_shifted_state.py,
pinned bit for bit to the three C oracles by tests/test_shifted_loop_reference.py.  The operation order is theirs; the
shifted SpMV is O.spmv followed by O.daxpy(sigma_seed, x, y).  Every per-shift update is one loop over the shifts of O.daxpy /
O.dscal calls, as in the oracles: a numpy expression across shifts would round differently.

exact=True evaluates every SpMV in long double and every dot product with math.fsum over the rounded products.  The distance
between the two evaluations is the rounding spread of the case itself.  Each state records the stop and switch decisions
taken so far, so that a test can tell whether both evaluations took the same ones."""
import math

import numpy as np

METHODS = ("shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab")
SCALARS = ("eta", "pi", "zeta", "alpha", "beta", "omega")     # per shift, in every state's "shift" dict


def _ops(O, n, ptr, col, val, exact):
    if exact:
        A = lambda x: O.spmv(n, ptr, col, val, x, long_double=True)
        dot = lambda x, y: math.fsum(x * y)
    else:
        A = lambda x: O.spmv(n, ptr, col, val, x)
        dot = O.ddot
    return A, dot


class _Keeper:
    """Collects the state after every wanted iteration; a wanted k past the end of the loop gets the state it ended in, which
    is what a solve with max_iter = k returns."""

    def __init__(self, ks, keep_p):
        self.want, self.keep_p, self.out, self.last = set(ks), keep_p, {}, None

    def __call__(self, k, ret, x, p, r, hist, seed, stop_iter, shift, decisions):
        st = dict(iters=k, ret=ret, x=x.copy(), r=r.copy(), p=p.copy() if self.keep_p else None, hist=np.array(hist),
                  seed=seed, stop_iter=stop_iter.copy(), shift={q: np.array(v) for q, v in shift.items()},
                  decisions=list(decisions))
        self.last = st
        if k in self.want:
            self.out[k] = st

    def done(self):
        for k in self.want:
            if k not in self.out and self.last is not None and self.last["iters"] < k:
                self.out[k] = self.last
        return self.out


def _switching(O, n, ptr, col, val, b, sigma, seed, tol, max_iter_opt, exact, keep, x0):
    """orc_shifted_lopbicg_switching (shifted_switching_solver.c:260-602)."""
    A, dot = _ops(O, n, ptr, col, val, exact)
    ax, sc = O.daxpy, O.dscal
    L = sigma.size
    x = np.zeros((L, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(L, n)
    r = b.copy()
    k, max_iter, stop_count, max_sigma = 1, max_iter_opt + 1, 0, seed
    rTr = dot(r, r)
    r_hat = r.copy()
    p = np.empty((L, n))
    p[:] = r
    alpha_set, beta_set, omega_set = np.ones(L), np.zeros(L), np.zeros(L)
    eta_set, zeta_set = np.zeros(L), np.ones(L)
    PI = np.zeros((L, max(max_iter, 2)))
    PI[:, 0] = PI[:, 1] = 1.0
    alpha_arch, beta_arch, omega_arch = np.zeros(max_iter + 1), np.zeros(max_iter + 1), np.zeros(max_iter + 1)
    alpha_arch[0], beta_arch[0] = 1.0, 0.0
    stop_flag = np.zeros(L, dtype=bool)
    stop_iter = np.zeros(L, dtype=np.int64)
    dot_r = dot_zero = rTr
    hist, decisions = [1.0], []
    while stop_count < L and k < max_iter:                               # :372
        r_old = r.copy()                                                 # :374
        s = A(p[seed]); ax(sigma[seed], p[seed], s)                      # :377-386
        rTs = dot(r_hat, s)
        alpha_arch[k] = rTr / rTs                                        # :390
        ax(-alpha_arch[k], s, r)                                         # :391  q
        q_copy = r.copy()                                                # :392
        y = A(r); ax(sigma[seed], r, y)                                  # :395-404
        qTq, qTy = dot(r, r), dot(r, y)
        omega_arch[k] = qTq / qTy                                        # :410
        ax(alpha_arch[k], p[seed], x[seed]); ax(omega_arch[k], r, x[seed])            # :411-412
        ax(-omega_arch[k], y, r)                                         # :413
        dot_r = dot(r, r)                                                # :414
        rTr_old = rTr
        rTr = dot(r_hat, r)                                              # :416
        beta_arch[k] = (alpha_arch[k] / omega_arch[k]) * (rTr / rTr_old)              # :420
        sc(beta_arch[k], p[seed]); ax(1.0, r, p[seed]); ax(-beta_arch[k] * omega_arch[k], s, p[seed])   # :421-423
        for j in range(L):                                               # :429-446
            if j == seed or stop_flag[j]:
                continue
            eta_set[j] = ((beta_arch[k - 1] / alpha_arch[k - 1]) * alpha_arch[k] * eta_set[j]
                          - (sigma[seed] - sigma[j]) * alpha_arch[k] * PI[j, k - 1])
            PI[j, k] = eta_set[j] + PI[j, k - 1]
            alpha_set[j] = (PI[j, k - 1] / PI[j, k]) * alpha_arch[k]
            omega_set[j] = omega_arch[k] / (1.0 - omega_arch[k] * (sigma[seed] - sigma[j]))
            ax(omega_set[j] / (PI[j, k] * zeta_set[j]), q_copy, x[j])
            ax(alpha_set[j], p[j], x[j])
            ax(omega_set[j] / (alpha_set[j] * zeta_set[j] * PI[j, k]), q_copy, p[j])
            ax(-omega_set[j] / (alpha_set[j] * zeta_set[j] * PI[j, k - 1]), r_old, p[j])
            zeta_set[j] = (1.0 - omega_arch[k] * (sigma[seed] - sigma[j])) * zeta_set[j]
            beta_set[j] = (PI[j, k - 1] / PI[j, k]) * (PI[j, k - 1] / PI[j, k]) * beta_arch[k]
            sc(beta_set[j], p[j])
            ax(1.0 / (PI[j, k] * zeta_set[j]), r, p[j])
        max_zeta_pi = 1.0                                                # :451-476
        for j in range(L):
            if stop_flag[j]:
                continue
            azp = 1.0 if j == seed else abs(1.0 / (zeta_set[j] * PI[j, k]))
            if azp * azp * dot_r <= tol * tol * dot_zero:
                stop_flag[j] = True; stop_count += 1; stop_iter[j] = k
                decisions.append(("stop", k, j))
            elif azp > max_zeta_pi:
                max_zeta_pi = azp; max_sigma = j
        if stop_flag[seed] and stop_count < L:                           # :490-527 seed switch
            ms = max_sigma
            for i in range(1, k + 1):
                alpha_arch[i] = (PI[ms, i - 1] / PI[ms, i]) * alpha_arch[i]
                beta_arch[i] = (PI[ms, i - 1] / PI[ms, i]) * (PI[ms, i - 1] / PI[ms, i]) * beta_arch[i]
                omega_arch[i] = omega_arch[i] / (1.0 - omega_arch[i] * (sigma[seed] - sigma[ms]))
            sc(1.0 / (zeta_set[ms] * PI[ms, k]), r)
            eta_set[:] = 0.0
            zeta_set[:] = 1.0
            for i in range(1, k + 1):
                for j in range(L):
                    if stop_flag[j] or j == ms:
                        continue
                    eta_set[j] = ((beta_arch[i - 1] / alpha_arch[i - 1]) * alpha_arch[i] * eta_set[j]
                                  - (sigma[ms] - sigma[j]) * alpha_arch[i] * PI[j, i - 1])
                    PI[j, i] = eta_set[j] + PI[j, i - 1]
                    zeta_set[j] = (1.0 - omega_arch[i] * (sigma[ms] - sigma[j])) * zeta_set[j]
            seed = ms
            decisions.append(("switch", k, ms))
        hist.append(dot_r / dot_zero)
        keep(k, k + 1, x, p, r, hist, seed, stop_iter,
             dict(eta=eta_set, pi=PI[:, k], zeta=zeta_set, alpha=alpha_set, beta=beta_set, omega=omega_set), decisions)
        k += 1                                                           # :537
    return k


def _fixed(O, n, ptr, col, val, b, sigma, seed, tol, max_iter, exact, keep, x0):
    """orc_shifted_lopbicg (shifted_switching_solver.c:20-257)."""
    A, dot = _ops(O, n, ptr, col, val, exact)
    ax, sc = O.daxpy, O.dscal
    L = sigma.size
    x = np.zeros((L, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(L, n)
    r = b.copy()
    k, stop_count = 0, 0
    sg = sigma[seed]
    rTr = dot(r, r)
    r_hat = r.copy()
    p = np.empty((L, n))
    p[:] = r
    alpha_set, beta_set, omega_set = np.ones(L), np.zeros(L), np.zeros(L)
    eta_set, zeta_set, pi_old, pi_new = np.zeros(L), np.ones(L), np.ones(L), np.ones(L)
    stop_flag = np.zeros(L, dtype=bool)
    stop_iter = np.zeros(L, dtype=np.int64)
    dot_r = dot_zero = rTr
    hist, decisions = [1.0], []
    while stop_count < L and k < max_iter:                               # :106
        r_old = r.copy()                                                 # :108
        pi_old[:] = pi_new                                               # :109
        alpha_old, beta_old = alpha_set[seed], beta_set[seed]            # :110-111
        s = A(p[seed]); ax(sg, p[seed], s)                               # :113-114
        rTs = dot(r_hat, s)
        alpha_set[seed] = rTr / rTs                                      # :119
        ax(-alpha_set[seed], s, r)                                       # :120  q
        y = A(r); ax(sg, r, y)                                           # :121-122
        qTq, qTy = dot(r, r), dot(r, y)
        omega_set[seed] = qTq / qTy                                      # :128
        ax(alpha_set[seed], p[seed], x[seed]); ax(omega_set[seed], r, x[seed])       # :129-130
        for j in range(L):                                               # :136-149
            if j == seed or stop_flag[j]:
                continue
            eta_set[j] = (beta_old / alpha_old) * alpha_set[seed] * eta_set[j] - (sigma[seed] - sigma[j]) * alpha_set[seed] * pi_old[j]
            pi_new[j] = eta_set[j] + pi_old[j]
            alpha_set[j] = (pi_old[j] / pi_new[j]) * alpha_set[seed]
            omega_set[j] = omega_set[seed] / (1.0 - omega_set[seed] * (sigma[seed] - sigma[j]))
            ax(omega_set[j] / (pi_new[j] * zeta_set[j]), r, x[j])
            ax(alpha_set[j], p[j], x[j])
            ax(omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_new[j]), r, p[j])
            ax(-omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_old[j]), r_old, p[j])
            zeta_set[j] = (1.0 - omega_set[seed] * (sigma[seed] - sigma[j])) * zeta_set[j]
        ax(-omega_set[seed], y, r)                                       # :156  r
        dot_r = dot(r, r)
        rTr_old = rTr
        rTr = dot(r_hat, r)
        beta_set[seed] = (alpha_set[seed] / omega_set[seed]) * (rTr / rTr_old)       # :163
        sc(beta_set[seed], p[seed]); ax(1.0, r, p[seed]); ax(-beta_set[seed] * omega_set[seed], s, p[seed])   # :164-166
        for j in range(L):                                               # :168-174
            if j == seed or stop_flag[j]:
                continue
            beta_set[j] = (pi_old[j] / pi_new[j]) * (pi_old[j] / pi_new[j]) * beta_set[seed]
            sc(beta_set[j], p[j])
            ax(1.0 / (pi_new[j] * zeta_set[j]), r, p[j])
        for j in range(L):                                               # :184-203
            if stop_flag[j]:
                continue
            azp = 1.0 if j == seed else abs(1.0 / (zeta_set[j] * pi_new[j]))
            if azp * azp * dot_r <= tol * tol * dot_zero:
                stop_flag[j] = True; stop_count += 1; stop_iter[j] = k + 1
                decisions.append(("stop", k + 1, j))
        k += 1                                                           # :214
        hist.append(dot_r / dot_zero)
        keep(k, k, x, p, r, hist, seed, stop_iter,
             dict(eta=eta_set, pi=pi_new, zeta=zeta_set, alpha=alpha_set, beta=beta_set, omega=omega_set), decisions)
    return k


def _lop(O, n, ptr, col, val, b, sigma, seed, tol, max_iter, exact, keep, x0, pipe):
    """orc_shifted_lop (shifted_solver.c:182-354 / :703-895)."""
    A, dot = _ops(O, n, ptr, col, val, exact)
    ax, sc = O.daxpy, O.dscal
    L = sigma.size
    x = np.zeros((L, n)) if x0 is None else np.array(x0, dtype=np.float64).reshape(L, n)
    r = b.copy()
    p = np.zeros((L, n))                                                 # p_loc_set = calloc (:226 / :748)
    s, y, z, w, v, t = (np.zeros(n) for _ in range(6))
    alpha_set, beta_set, omega_set = np.ones(L), np.zeros(L), np.zeros(L)
    eta_set, zeta_set, pi_old, pi_new = np.zeros(L), np.ones(L), np.ones(L), np.ones(L)
    alpha_old = beta_old = rTs = rTw = qTq = wTw = 0.0
    sg = sigma[seed]
    k = 0
    rTr = dot(r, r)                                                      # :240 / :763
    if pipe:
        w = A(r); ax(sg, r, w)                                           # :765-766
        rTw = dot(r, w)
        t = A(w); ax(sg, w, t)                                           # :769-770
    r_hat = r.copy()
    p[seed] = r                                                          # :252 / :782
    if pipe:
        alpha_old = 1.0; alpha_set[seed] = rTr / rTw                     # :786-787
    dot_r = dot_zero = rTr
    max_zeta_pi = 1.0
    hist, decisions = [1.0], []
    stop_iter = np.zeros(L, dtype=np.int64)
    while True:
        if not max_zeta_pi * max_zeta_pi * dot_r > tol * tol * dot_zero:     # :259 / :793
            decisions.append(("converged", k))
            break
        if not k < max_iter:
            break
        if not pipe:
            s = A(p[seed]); ax(sg, p[seed], s)                           # :261-262
            rTs = dot(r_hat, s)
        else:
            ax(-omega_set[seed], s, p[seed]); sc(beta_set[seed], p[seed]); ax(1.0, r, p[seed])   # :795-797
            ax(-omega_set[seed], z, s); sc(beta_set[seed], s); ax(1.0, w, s)                     # :798-800
            ax(-omega_set[seed], v, z); sc(beta_set[seed], z); ax(1.0, t, z)                     # :801-803
        for j in range(L):                                               # :264-269 / :804-809
            if j == seed:
                continue
            beta_set[j] = (pi_old[j] / pi_new[j]) * (pi_old[j] / pi_new[j]) * beta_set[seed]
            sc(beta_set[j], p[j])
            ax(1.0 / (pi_new[j] * zeta_set[j]), r, p[j])
        if not pipe:
            pi_old[:] = pi_new                                           # :270
            r_old = r.copy()
            alpha_old, beta_old = alpha_set[seed], beta_set[seed]
            alpha_set[seed] = rTr / rTs                                  # :276
            ax(-alpha_set[seed], s, r)                                   # :277  q
            y = A(r); ax(sg, r, y)                                       # :278-279
            qTq, qTy = dot(r, r), dot(r, y)
        else:
            r_old = r.copy()                                             # :810
            ax(-alpha_set[seed], s, r)                                   # :811  q
            ax(-alpha_set[seed], z, w)                                   # :812  y (in w)
            qTy, wTw = dot(r, w), dot(w, w)
            v = A(z); ax(sg, z, v)                                       # :815-816
            pi_old[:] = pi_new                                           # :817
            beta_old = beta_set[seed]
        for j in range(L):                                               # :283-289 / :819-825
            if j == seed:
                continue
            eta_set[j] = (beta_old / alpha_old) * alpha_set[seed] * eta_set[j] - (sigma[seed] - sigma[j]) * alpha_set[seed] * pi_old[j]
            pi_new[j] = eta_set[j] + pi_old[j]
            alpha_set[j] = (pi_old[j] / pi_new[j]) * alpha_set[seed]
        omega_set[seed] = qTy / wTw if pipe else qTq / qTy               # :293 / :829
        ax(alpha_set[seed], p[seed], x[seed]); ax(omega_set[seed], r, x[seed])       # :294-295 / :830-831
        for j in range(L):                                               # :296-304 / :832-840
            if j == seed:
                continue
            omega_set[j] = omega_set[seed] / (1.0 - omega_set[seed] * (sigma[seed] - sigma[j]))
            ax(omega_set[j] / (pi_new[j] * zeta_set[j]), r, x[j])
            ax(alpha_set[j], p[j], x[j])
            ax(omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_new[j]), r, p[j])
            ax(-omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_old[j]), r_old, p[j])
            zeta_set[j] = (1.0 - omega_set[seed] * (sigma[seed] - sigma[j])) * zeta_set[j]
        if not pipe:
            ax(-omega_set[seed], y, r)                                   # :305  r
            dot_r = dot(r, r)
            rTr_old = rTr
            rTr = dot(r_hat, r)
            beta_set[seed] = (alpha_set[seed] / omega_set[seed]) * (rTr / rTr_old)   # :312
        else:
            ax(-omega_set[seed], w, r)                                   # :841  r
            dot_r = dot(r, r)
            ax(-alpha_set[seed], v, t)                                   # :843
            ax(-omega_set[seed], t, w)                                   # :844  w
            rTr_old = rTr
            rTr, rTw, rTs, rTz = dot(r_hat, r), dot(r_hat, w), dot(r_hat, s), dot(r_hat, z)
            t = A(w); ax(sg, w, t)                                       # :850-851
            beta_set[seed] = (alpha_set[seed] / omega_set[seed]) * (rTr / rTr_old)   # :857
            alpha_old = alpha_set[seed]
            alpha_set[seed] = rTr / (rTw + beta_set[seed] * (rTs - omega_set[seed] * rTz))   # :859
        max_zeta_pi = 1.0                                                # :313-318 / :860-865
        for j in range(L):
            if j == seed:
                continue
            azp = abs(1.0 / (zeta_set[j] * pi_new[j]))
            if azp > max_zeta_pi:
                max_zeta_pi = azp
        if not pipe:
            sc(beta_set[seed], p[seed]); ax(1.0, r, p[seed]); ax(-beta_set[seed] * omega_set[seed], s, p[seed])   # :319-321
        k += 1                                                           # :323 / :867
        hist.append(dot_r / dot_zero)
        keep(k, k, x, p, r, hist, seed, stop_iter,
             dict(eta=eta_set, pi=pi_new, zeta=zeta_set, alpha=alpha_set, beta=beta_set, omega=omega_set), decisions)
    return k


def _run(O, method, ptr, col, val, b, sigma, seed, ks, tol, exact, keep_p, x0=None):
    b = np.ascontiguousarray(b, dtype=np.float64)
    n = b.size
    ptr = np.ascontiguousarray(ptr, dtype=np.uint32)
    col = np.ascontiguousarray(col, dtype=np.uint32)
    val = np.ascontiguousarray(val, dtype=np.float64)
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    keep = _Keeper(ks, keep_p)
    args = (O, n, ptr, col, val, b, sigma, int(seed), float(tol), max(ks), exact, keep, x0)
    if method == "shifted_lopbicg_switching":
        ret = _switching(*args)
    elif method == "shifted_lopbicg":
        ret = _fixed(*args)
    elif method in ("shifted_lopbicgstab", "shifted_pipe_lopbicgstab"):
        ret = _lop(*args, pipe=method == "shifted_pipe_lopbicgstab")
    else:
        raise ValueError(method)
    return keep.done(), keep.last, ret


def shifted_reference_states(O, method, ptr, col, val, b, sigma, seed, ks, tol=0.0, exact=False, keep_p=True, x0=None):
    """The state after iteration k of `method` for every k in ks, in one pass: {k: state}, the state of a solve with
    max_iter = k (the state the loop ends in, if its tolerance test ends it first).  A state holds
      iters, ret          iterations performed and the solver's return value (switching: iterations + 1)
      x, p                (sigma_len, n): every x_j and p_j (p: None unless keep_p)
      r, hist             the seed residual and dot_r / dot_zero after iterations 0 .. iters
      seed, stop_iter     the seed after the last iteration, the iteration at which every shift stopped (0: never)
      shift               per-shift scalars of the last iteration (SCALARS)
      decisions           every stop / switch decision so far: ("stop", k, j), ("switch", k, new seed), ("converged", k)
    x0 (sigma_len, n) is the initial x_set (None: zero).  None of the four solvers forms b - A x0: r starts at b whatever x0 is,
    and each x_j only ever has corrections added to it."""
    return _run(O, method, ptr, col, val, b, sigma, seed, ks, tol, exact, keep_p, x0)[0]


def shifted_reference_solve(O, method, ptr, col, val, b, sigma, seed, tol, max_iter, keep_p=False, x0=None):
    """The whole solve: (the state it ends in, the solver's return value)."""
    _, last, k = _run(O, method, ptr, col, val, b, sigma, seed, [max_iter], tol, False, keep_p, x0)
    return last, (k if method == "shifted_lopbicg_switching" else last["ret"] if last else 0)
