/*
 * shifted_lop_oracle.c -- CPU restatement of the LOP family of the reference's shifted_solver.h (shifted_lopbicgstab and
 * shifted_pipe_lopbicgstab, shifted_solver.c:182-354, 703-895).  TEST INFRASTRUCTURE ONLY, like bicg_oracle.c: only tests/
 * load it, as the checker; the product never links or calls it.
 *
 * It includes bicg_oracle.c so that it uses the same P-rank emulation of the SpMV and of the dot products (orc_sys,
 * orc_spmv_sys, orc_dot) and the same BLAS-1 restatements of vector.c, not a second copy of them; the result is a library of
 * its own (liboracle_lop.so, recipe oracle/shifted_lop.mk).  Parity pin: tests/test_oracle_golden_shifted_lop.py requires
 * bit-identical output against the reference's own shifted_solver.c compiled in place (golden data in tests/golden/).
 */
#include "bicg_oracle.c"


/* ---- shifted_lopbicgstab / shifted_pipe_lopbicgstab: shifted_solver.c:182-354, 703-895 --------------------------------
 * Shifted BiCGStab without seed switching: the seed system (A + sigma[seed] I) x = b is iterated with BiCGStab (LOP) or with
 * the pipelined recurrences of pipe_bicgstab (PIPE-LOP); every other shift is advanced from the seed's Krylov data in every
 * iteration until max_zeta_pi^2 dot_r <= tol^2 dot_zero or max_iter.  Restated line by line (the _v2 / _nooverlap twins of
 * the reference are the same arithmetic); P-rank emulation of the dots and of the SpMV as in bicg_oracle.c.  x_set: sigma_len blocks of
 * n (added to), r: b in, seed residual out.  Returns k, the iterations performed; hist[k] = dot_r / dot_zero after iteration
 * k.  PIPE-LOP reads omega[seed] and s, z, v before writing them in its first iteration (:795-803): they start at 0 here. */
static int orc_shifted_lop(int n, const double *val, const unsigned *col, const unsigned *ptr, int P, double *x_set, double *r,
                           const double *sigma, int sigma_len, int seed, int pipe, double tol, int max_iter, double *hist,
                           int hist_cap)
{
    orc_sys S; orc_sys_init(&S, n, val, col, ptr, P);
    orc_opts o = { tol, max_iter, hist, hist_cap };
    int j, k = 0;
    double *r_old = vnew(n), *r_hat = vnew(n), *s = vnew(n), *y = vnew(n), *z = vnew(n), *w = vnew(n), *v = vnew(n), *t = vnew(n);
    double *p_set = (double *)calloc((size_t)n * (size_t)sigma_len, sizeof(double));            /* :226 / :748 */
    double *alpha_set = vnew(sigma_len), *beta_set = vnew(sigma_len), *omega_set = vnew(sigma_len), *eta_set = vnew(sigma_len),
           *zeta_set = vnew(sigma_len), *pi_old_set = vnew(sigma_len), *pi_new_set = vnew(sigma_len);
    double alpha_old = 0.0, beta_old = 0.0, dot_r, dot_zero, rTr, rTs = 0.0, rTw = 0.0, rTz, qTq = 0.0, qTy, wTw = 0.0, rTr_old, max_zeta_pi,
           abs_zeta_pi;
    const double sg = sigma[seed];
#define PSET(jj) (p_set + (size_t)(jj) * (size_t)n)
#define XSET(jj) (x_set + (size_t)(jj) * (size_t)n)

    rTr = orc_dot(&S, r, r);                                            /* :240 / :763 */
    if (pipe) {
        orc_spmv_sys(&S, r, w); orc_axpy(n, sg, r, w);                  /* :765-766 */
        rTw = orc_dot(&S, r, w);                                        /* :767 */
        orc_spmv_sys(&S, w, t); orc_axpy(n, sg, w, t);                  /* :769-770 */
    }
    orc_copy(n, r, r_hat);                                              /* :242 / :772 */
    for (j = 0; j < sigma_len; j++) {                                   /* :243-251 / :773-781 */
        beta_set[j] = 0.0; alpha_set[j] = 1.0; eta_set[j] = 0.0;
        pi_old_set[j] = 1.0; pi_new_set[j] = 1.0; zeta_set[j] = 1.0;
    }
    orc_copy(n, r, PSET(seed));                                         /* :252 / :782 */
    if (pipe) { alpha_old = 1.0; alpha_set[seed] = rTr / rTw; }        /* :786-787 */
    dot_r = rTr; dot_zero = rTr; max_zeta_pi = 1.0;                     /* :255-257 / :788-790 */
    hist_put(&o, 0, dot_r, dot_zero);

    while (max_zeta_pi * max_zeta_pi * dot_r > tol * tol * dot_zero && k < max_iter) {        /* :259 / :793 */
        if (!pipe) {
            orc_spmv_sys(&S, PSET(seed), s); orc_axpy(n, sg, PSET(seed), s);                  /* :261-262 */
            rTs = orc_dot(&S, r_hat, s);                                                      /* :263 */
        } else {
            orc_axpy(n, -omega_set[seed], s, PSET(seed)); orc_scal(n, beta_set[seed], PSET(seed)); orc_axpy(n, 1.0, r, PSET(seed));  /* :795-797 */
            orc_axpy(n, -omega_set[seed], z, s); orc_scal(n, beta_set[seed], s); orc_axpy(n, 1.0, w, s);                          /* :798-800 */
            orc_axpy(n, -omega_set[seed], v, z); orc_scal(n, beta_set[seed], z); orc_axpy(n, 1.0, t, z);                          /* :801-803 */
        }
        for (j = 0; j < sigma_len; j++) {                                                     /* :264-269 / :804-809 */
            if (j == seed) continue;
            beta_set[j] = (pi_old_set[j] / pi_new_set[j]) * (pi_old_set[j] / pi_new_set[j]) * beta_set[seed];
            orc_scal(n, beta_set[j], PSET(j));
            orc_axpy(n, 1.0 / (pi_new_set[j] * zeta_set[j]), r, PSET(j));
        }
        if (!pipe) {
            orc_copy(sigma_len, pi_new_set, pi_old_set);                                      /* :270 */
            orc_copy(n, r, r_old);                                                            /* :271 */
            alpha_old = alpha_set[seed]; beta_old = beta_set[seed];                           /* :272-273 */
            alpha_set[seed] = rTr / rTs;                                                      /* :276 */
            orc_axpy(n, -alpha_set[seed], s, r);                                              /* :277  q */
            orc_spmv_sys(&S, r, y); orc_axpy(n, sg, r, y);                                    /* :278-279 */
            qTq = orc_dot(&S, r, r);                                                          /* :281 */
            qTy = orc_dot(&S, r, y);                                                          /* :282 */
        } else {
            orc_copy(n, r, r_old);                                                            /* :810 */
            orc_axpy(n, -alpha_set[seed], s, r);                                              /* :811  q */
            orc_axpy(n, -alpha_set[seed], z, w);                                              /* :812  y (in w) */
            qTy = orc_dot(&S, r, w);                                                          /* :813 */
            wTw = orc_dot(&S, w, w);                                                          /* :814 */
            orc_spmv_sys(&S, z, v); orc_axpy(n, sg, z, v);                                    /* :815-816 */
            orc_copy(sigma_len, pi_new_set, pi_old_set);                                      /* :817 */
            beta_old = beta_set[seed];                                                        /* :818 */
        }
        for (j = 0; j < sigma_len; j++) {                                                     /* :283-289 / :819-825 */
            if (j == seed) continue;
            eta_set[j] = (beta_old / alpha_old) * alpha_set[seed] * eta_set[j] - (sigma[seed] - sigma[j]) * alpha_set[seed] * pi_old_set[j];
            pi_new_set[j] = eta_set[j] + pi_old_set[j];
            alpha_set[j] = (pi_old_set[j] / pi_new_set[j]) * alpha_set[seed];
        }
        omega_set[seed] = pipe ? qTy / wTw : qTq / qTy;                                       /* :293 / :829 */
        orc_axpy(n, alpha_set[seed], PSET(seed), XSET(seed));                                 /* :294 / :830 */
        orc_axpy(n, omega_set[seed], r, XSET(seed));                                          /* :295 / :831 */
        for (j = 0; j < sigma_len; j++) {                                                     /* :296-304 / :832-840 */
            if (j == seed) continue;
            omega_set[j] = omega_set[seed] / (1.0 - omega_set[seed] * (sigma[seed] - sigma[j]));
            orc_axpy(n, omega_set[j] / (pi_new_set[j] * zeta_set[j]), r, XSET(j));
            orc_axpy(n, alpha_set[j], PSET(j), XSET(j));
            orc_axpy(n, omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_new_set[j]), r, PSET(j));
            orc_axpy(n, -omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_old_set[j]), r_old, PSET(j));
            zeta_set[j] = (1.0 - omega_set[seed] * (sigma[seed] - sigma[j])) * zeta_set[j];
        }
        if (!pipe) {
            orc_axpy(n, -omega_set[seed], y, r);                                              /* :305  r */
            dot_r = orc_dot(&S, r, r);                                                        /* :306 */
            rTr_old = rTr;                                                                    /* :307 */
            rTr = orc_dot(&S, r_hat, r);                                                      /* :308 */
            beta_set[seed] = (alpha_set[seed] / omega_set[seed]) * (rTr / rTr_old);           /* :312 */
        } else {
            orc_axpy(n, -omega_set[seed], w, r);                                              /* :841  r */
            dot_r = orc_dot(&S, r, r);                                                        /* :842 */
            orc_axpy(n, -alpha_set[seed], v, t);                                              /* :843 */
            orc_axpy(n, -omega_set[seed], t, w);                                              /* :844  w */
            rTr_old = rTr;                                                                    /* :845 */
            rTr = orc_dot(&S, r_hat, r);                                                      /* :846 */
            rTw = orc_dot(&S, r_hat, w);                                                      /* :847 */
            rTs = orc_dot(&S, r_hat, s);                                                      /* :848 */
            rTz = orc_dot(&S, r_hat, z);                                                      /* :849 */
            orc_spmv_sys(&S, w, t); orc_axpy(n, sg, w, t);                                    /* :850-851 */
            beta_set[seed] = (alpha_set[seed] / omega_set[seed]) * (rTr / rTr_old);           /* :857 */
            alpha_old = alpha_set[seed];                                                      /* :858 */
            alpha_set[seed] = rTr / (rTw + beta_set[seed] * (rTs - omega_set[seed] * rTz));   /* :859 */
        }
        max_zeta_pi = 1.0;                                                                    /* :313-318 / :860-865 */
        for (j = 0; j < sigma_len; j++) {
            if (j == seed) continue;
            abs_zeta_pi = fabs(1.0 / (zeta_set[j] * pi_new_set[j]));
            if (abs_zeta_pi > max_zeta_pi) max_zeta_pi = abs_zeta_pi;
        }
        if (!pipe) {
            orc_scal(n, beta_set[seed], PSET(seed));                                          /* :319-321 */
            orc_axpy(n, 1.0, r, PSET(seed));
            orc_axpy(n, -beta_set[seed] * omega_set[seed], s, PSET(seed));
        }
        k++;                                                                                  /* :323 / :867 */
        hist_put(&o, k, dot_r, dot_zero);
    }
    free(r_old); free(r_hat); free(s); free(y); free(z); free(w); free(v); free(t); free(p_set);
    free(alpha_set); free(beta_set); free(omega_set); free(eta_set); free(zeta_set); free(pi_old_set); free(pi_new_set);
    orc_sys_free(&S);
#undef PSET
#undef XSET
    return k;
}

int orc_shifted_lopbicgstab(int n, const double *val, const unsigned *col, const unsigned *ptr, int P, double *x_set, double *r,
                            const double *sigma, int sigma_len, int seed, double tol, int max_iter, double *hist, int hist_cap)
{
    return orc_shifted_lop(n, val, col, ptr, P, x_set, r, sigma, sigma_len, seed, 0, tol, max_iter, hist, hist_cap);
}

int orc_shifted_pipe_lopbicgstab(int n, const double *val, const unsigned *col, const unsigned *ptr, int P, double *x_set,
                                 double *r, const double *sigma, int sigma_len, int seed, double tol, int max_iter, double *hist,
                                 int hist_cap)
{
    return orc_shifted_lop(n, val, col, ptr, P, x_set, r, sigma, sigma_len, seed, 1, tol, max_iter, hist, hist_cap);
}
