/*
 * shifted_fixed_oracle.c -- CPU restatement of shifted_lopbicg, the fixed-seed shifted LOP-BiCG of the reference's
 * shifted_switching_solver.h:11 (shifted_switching_solver.c:20-257).  TEST INFRASTRUCTURE ONLY, like bicg_oracle.c: only tests/
 * load it, as the checker; the product never links or calls it.
 *
 * It includes bicg_oracle.c so that it uses the same P-rank emulation of the SpMV and of the dot products (orc_sys,
 * orc_spmv_sys, orc_dot) and the same BLAS-1 restatements of vector.c, not a second copy of them; the result is a library of
 * its own (liboracle_fixed.so, recipe oracle/shifted_fixed.mk).  Parity pin: tests/test_oracle_golden_shifted_fixed.py requires
 * bit-identical output against the reference's own shifted_switching_solver.c compiled in place (golden data in tests/golden/).
 */
#include "bicg_oracle.c"


/* ---- shifted_lopbicg: shifted_switching_solver.c:20-257 ------------------------------------------------------------------
 * The seed system (A + sigma[seed] I) x = b is iterated with BiCGStab; every other shift j is advanced from the seed's Krylov
 * data with the collinear-residual recurrences (eta, pi, zeta) of the switching solver, and stops on its own once
 * |1/(zeta_j pi_j)|^2 dot_r <= tol^2 dot_zero.  The seed never changes: when it converges first its stop flag is set and
 * counted, but its BiCGStab keeps running (the shifts still need its Krylov data) until every shift has stopped or max_iter.
 * Restated line by line in the reference's order; P-rank emulation of the dots and of the SpMV as in bicg_oracle.c.
 * x_set: sigma_len blocks of n (added to), r: b in, seed residual out.  Returns k, the iterations performed (:255);
 * hist[k] = dot_r / dot_zero after iteration k (hist[0] = 1); stop_iter[j] = the iteration (1-based) after which shift j
 * stopped, 0 if it never did.  EPS 1e-12, MAX_ITER 1000 in the reference (:5-6). */
int orc_shifted_lopbicg(int n, const double *val, const unsigned *col, const unsigned *ptr, int P, double *x_set, double *r,
                        const double *sigma, int sigma_len, int seed, double tol, int max_iter, double *hist, int hist_cap,
                        int *stop_iter)
{
    orc_sys S; orc_sys_init(&S, n, val, col, ptr, P);
    orc_opts o = { tol, max_iter, hist, hist_cap };
    int j, k = 0, stop_count = 0;                                       /* :53-56 */
    double *r_old = vnew(n), *r_hat = vnew(n), *s = vnew(n), *y = vnew(n);
    double *p_set = (double *)calloc((size_t)n * (size_t)sigma_len, sizeof(double));            /* :65 */
    double *alpha_set = vnew(sigma_len), *beta_set = vnew(sigma_len), *omega_set = vnew(sigma_len), *eta_set = vnew(sigma_len),
           *zeta_set = vnew(sigma_len), *pi_old_set = vnew(sigma_len), *pi_new_set = vnew(sigma_len);
    char *stop_flag = (char *)calloc((size_t)sigma_len, 1);                                    /* :75 */
    double alpha_old, beta_old, dot_r, dot_zero, rTr, rTs, qTq, qTy, rTr_old, abs_zeta_pi;
    const double sg = sigma[seed];
#define PSET(jj) (p_set + (size_t)(jj) * (size_t)n)
#define XSET(jj) (x_set + (size_t)(jj) * (size_t)n)

    rTr = orc_dot(&S, r, r);                                            /* :83 */
    orc_copy(n, r, r_hat);                                              /* :85 */
    for (j = 0; j < sigma_len; j++) {                                   /* :86-94 */
        orc_copy(n, r, PSET(j));
        alpha_set[j] = 1.0; beta_set[j] = 0.0; eta_set[j] = 0.0;
        pi_old_set[j] = 1.0; pi_new_set[j] = 1.0; zeta_set[j] = 1.0;
    }
    orc_copy(n, r, PSET(seed));                                         /* :95 */
    dot_r = rTr; dot_zero = rTr;                                        /* :98-99 */
    hist_put(&o, 0, dot_r, dot_zero);
    if (stop_iter) for (j = 0; j < sigma_len; j++) stop_iter[j] = 0;

    while (stop_count < sigma_len && k < max_iter) {                    /* :106 */
        orc_copy(n, r, r_old);                                          /* :108 */
        orc_copy(sigma_len, pi_new_set, pi_old_set);                    /* :109 */
        alpha_old = alpha_set[seed]; beta_old = beta_set[seed];         /* :110-111 */
        orc_spmv_sys(&S, PSET(seed), s); orc_axpy(n, sg, PSET(seed), s);                      /* :113-114 */
        rTs = orc_dot(&S, r_hat, s);                                                          /* :116 */
        alpha_set[seed] = rTr / rTs;                                                          /* :119 */
        orc_axpy(n, -alpha_set[seed], s, r);                                                  /* :120  q */
        orc_spmv_sys(&S, r, y); orc_axpy(n, sg, r, y);                                        /* :121-122 */
        qTq = orc_dot(&S, r, r);                                                              /* :123 */
        qTy = orc_dot(&S, r, y);                                                              /* :124 */
        omega_set[seed] = qTq / qTy;                                                          /* :128 */
        orc_axpy(n, alpha_set[seed], PSET(seed), XSET(seed));                                 /* :129 */
        orc_axpy(n, omega_set[seed], r, XSET(seed));                                          /* :130 */
        for (j = 0; j < sigma_len; j++) {                                                     /* :136-149 */
            if (j == seed) continue;
            if (stop_flag[j]) continue;
            eta_set[j] = (beta_old / alpha_old) * alpha_set[seed] * eta_set[j] - (sigma[seed] - sigma[j]) * alpha_set[seed] * pi_old_set[j];
            pi_new_set[j] = eta_set[j] + pi_old_set[j];
            alpha_set[j] = (pi_old_set[j] / pi_new_set[j]) * alpha_set[seed];
            omega_set[j] = omega_set[seed] / (1.0 - omega_set[seed] * (sigma[seed] - sigma[j]));
            orc_axpy(n, omega_set[j] / (pi_new_set[j] * zeta_set[j]), r, XSET(j));
            orc_axpy(n, alpha_set[j], PSET(j), XSET(j));
            orc_axpy(n, omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_new_set[j]), r, PSET(j));
            orc_axpy(n, -omega_set[j] / (alpha_set[j] * zeta_set[j] * pi_old_set[j]), r_old, PSET(j));
            zeta_set[j] = (1.0 - omega_set[seed] * (sigma[seed] - sigma[j])) * zeta_set[j];
        }
        orc_axpy(n, -omega_set[seed], y, r);                                                  /* :156  r */
        dot_r = orc_dot(&S, r, r);                                                            /* :157 */
        rTr_old = rTr;                                                                        /* :158 */
        rTr = orc_dot(&S, r_hat, r);                                                          /* :159 */
        beta_set[seed] = (alpha_set[seed] / omega_set[seed]) * (rTr / rTr_old);               /* :163 */
        orc_scal(n, beta_set[seed], PSET(seed));                                              /* :164-166 */
        orc_axpy(n, 1.0, r, PSET(seed));
        orc_axpy(n, -beta_set[seed] * omega_set[seed], s, PSET(seed));
        for (j = 0; j < sigma_len; j++) {                                                     /* :168-174 */
            if (j == seed) continue;
            if (stop_flag[j]) continue;
            beta_set[j] = (pi_old_set[j] / pi_new_set[j]) * (pi_old_set[j] / pi_new_set[j]) * beta_set[seed];
            orc_scal(n, beta_set[j], PSET(j));
            orc_axpy(n, 1.0 / (pi_new_set[j] * zeta_set[j]), r, PSET(j));
        }
        for (j = 0; j < sigma_len; j++) {                                                     /* :184-203 */
            if (stop_flag[j]) continue;
            if (j == seed) abs_zeta_pi = 1.0;
            else abs_zeta_pi = fabs(1.0 / (zeta_set[j] * pi_new_set[j]));
            if (abs_zeta_pi * abs_zeta_pi * dot_r <= tol * tol * dot_zero) {
                stop_flag[j] = 1; stop_count++;
                if (stop_iter) stop_iter[j] = k + 1;
            }
        }
        k++;                                                                                  /* :214 */
        hist_put(&o, k, dot_r, dot_zero);
    }
    free(r_old); free(r_hat); free(s); free(y); free(p_set);
    free(alpha_set); free(beta_set); free(omega_set); free(eta_set); free(zeta_set); free(pi_old_set); free(pi_new_set);
    free(stop_flag);
    orc_sys_free(&S);
#undef PSET
#undef XSET
    return k;                                                           /* :255 */
}
