// shifted.cu -- shifted_lopbicg_switching (shifted_switching_solver.c:260-602; prototype shifted_switching_solver.h:12):
// seed-switching shifted BiCGStab for (A + sigma_j I) x_j = b, j = 0 .. sigma_len - 1, behind the reference's own entry point.
//
// One seed system is iterated with BiCGStab on the arena vectors with the same fused SpMV (+ sigma_seed x in the
// epilogue) and reduction tails as the un-shifted solvers; every other shift is advanced from the seed's Krylov data:
//   * the per-shift scalar recurrences (eta, pi, zeta, alpha_j, omega_j, beta_j; :431-445; all but beta_j through
//     shift_step of shifted_run.cuh), the convergence tests (:451-476) and the seed switch (:490-527, history of alpha /
//     beta / omega / pi re-derived for the new seed) run in ONE small kernel per iteration (sh_scalar_iter), entirely on
//     the device;
//   * the six daxpy / dscal passes per shift and iteration of the reference (:435-445: up to 512 shifts x 6 passes over
//     length-n vectors) are ONE multi-vector kernel (sh_vec_shift): q, r_old and r are loaded once per row, then x_j and
//     p_j of every active shift are read and written exactly once -- 32 B per row and shift, the HBM floor of the method.
// Element-wise operation order = the reference's call order with gcc's FMA contraction (y += a x -> fma(a, x, y)).
// The host only enqueues: the loop runs on the device as a CUDA graph WHILE node (as solve.cu's kernel-per-phase loop does).
//
// The same solve also runs shifted_lopbicg (shifted_switching_solver.c:20-257; prototype :11), the fixed-seed variant: until the
// seed converges its arithmetic is the switching solver's line for line.  With ShiftDev::fixed set, sh_scalar_iter skips the
// seed switch, so a seed that converges first is counted as stopped but its BiCGStab keeps running (the other shifts still
// advance from its Krylov data) until every shift has stopped or MAX_ITER.  It returns the iterations performed, not + 1,
// and prints only the two MEASURE_TIME lines (:241-242).
#include "engine.hpp"
#include "shifted_run.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace bicg {

namespace {

constexpr int SH_COEF = 6;          // per active shift: c1, alpha_j, c2, c3, beta_j, c4
constexpr size_t SH_ENTRY = SH_COEF * sizeof(double) + sizeof(int);     // shared memory of sh_vec_shift per shift: coefficients, index
constexpr int SH_EVENTS = 16;       // seed switches remembered for the reference's printf lines

struct ShiftDev {
    int L, max_iter;                // sigma_len, MAX_ITER + 1                                    (:291-293)
    int fixed;                      // 1: shifted_lopbicg, the seed never switches               (:20-257)
    double tol;                     // EPS                                                       (:292)
    int seed, k, stop_count, done, live, switched, max_sigma, n_active, n_events;
    double rTr, rTs, qTq, qTy, dot_r, dot_zero, rTr_old, r_scale;
    double sigma_seed;              // read by the SpMV epilogue
    double *sigma, *alpha_set, *beta_set, *omega_set, *eta_set, *zeta_set;      // [L]
    unsigned char *stop_flag;                                                  // [L]
    int *stop_iter;                                                             // [L]
    double *alpha_arch, *beta_arch, *omega_arch;                                // [max_iter]
    double *pi_arch;                                                            // [L][max_iter]
    double *coef;                                                               // [L][SH_COEF], compacted with `active`
    int *active;                                                                // [L]
    double *hist;                                                               // [max_iter + 1]
    int *ev_k, *ev_seed, *ev_remain;                                            // [SH_EVENTS]
    double *ev_vals;                                                            // [SH_EVENTS][L][3]  eta, pi, zeta (:518)
};

#define PI(j, kk) sd->pi_arch[(size_t)(j) * (size_t)sd->max_iter + (size_t)(kk)]

// ---- scalar kernels ------------------------------------------------------------------------------------------------
__global__ void sh_scalar_init(ShiftDev *sd, Scalars *sc)                           // :342-362
{
    const int t = threadIdx.x;
    if (t == 0) {
        sd->rTr = sc->pend[0]; sd->dot_r = sd->rTr; sd->dot_zero = sd->rTr;
        sd->k = 1; sd->stop_count = 0; sd->done = 0; sd->live = 0; sd->switched = 0; sd->n_events = 0; sd->max_sigma = sd->seed;
        sd->alpha_arch[0] = 1.0; sd->beta_arch[0] = 0.0;
        sd->sigma_seed = sd->sigma[sd->seed];
        sd->hist[0] = 1.0;
        if (!(sd->k < sd->max_iter) || sd->L <= 0) sd->done = 1;
    }
    for (int j = t; j < sd->L; j += blockDim.x) {
        sd->alpha_set[j] = 1.0; sd->beta_set[j] = 0.0; sd->eta_set[j] = 0.0; sd->zeta_set[j] = 1.0;
        PI(j, 0) = 1.0; PI(j, 1) = 1.0;
        sd->stop_flag[j] = 0; sd->stop_iter[j] = 0;
    }
}
__global__ void sh_scalar_alpha(ShiftDev *sd, Scalars *sc)                          // :387-390
{
    sd->live = !sd->done;
    if (sd->done) return;
    sd->switched = 0;
    sd->rTs = sc->pend[0];
    const double al = sd->rTr / sd->rTs;
    sd->alpha_arch[sd->k] = al;
    sc->alpha = al;
}
__global__ void sh_scalar_omega(ShiftDev *sd, Scalars *sc)                          // :405-410
{
    if (sd->done) return;
    sd->qTq = sc->pend[0]; sd->qTy = sc->pend[1];
    const double om = sd->qTq / sd->qTy;
    sd->omega_arch[sd->k] = om;
    sc->omega = om;
}
// beta, the shifts' recurrences, convergence tests, seed switch, loop test: one block
__global__ void __launch_bounds__(512) sh_scalar_iter(ShiftDev *sd, Scalars *sc)
{
    if (sd->done) return;
    const int t = threadIdx.x, T = blockDim.x;
    const int k = sd->k, L = sd->L;
    __shared__ int s_n;
    if (t == 0) {
        sd->dot_r = sc->pend[0];                                                    // :414
        sd->rTr_old = sd->rTr;                                                      // :415
        sd->rTr = sc->pend[1];                                                      // :416
        const double be = (sd->alpha_arch[k] / sd->omega_arch[k]) * (sd->rTr / sd->rTr_old);      // :420
        sd->beta_arch[k] = be;
        sc->beta = be;
        s_n = 0;
    }
    __syncthreads();
    const int seed = sd->seed;
    const double al_k = sd->alpha_arch[k], om_k = sd->omega_arch[k], be_k = sd->beta_arch[k];
    const double al_o = sd->alpha_arch[k - 1], be_o = sd->beta_arch[k - 1], sg_s = sd->sigma[seed];
    for (int j = t; j < L; j += T) {                                                // :429-446 (scalars; vectors: sh_vec_shift)
        if (j == seed || sd->stop_flag[j]) continue;
        const double pi_o = PI(j, k - 1);
        const ShiftStep u = shift_step(al_k, al_o, be_o, om_k, sg_s - sd->sigma[j], sd->eta_set[j], pi_o, sd->zeta_set[j]);
        // p_j is scaled at the end of this iteration, so with this iteration's beta, pi and zeta (:442-445)
        const double be_j = (pi_o / u.pi) * (pi_o / u.pi) * be_k;
        const double c4 = 1.0 / (u.pi * u.zeta);
        sd->eta_set[j] = u.eta; PI(j, k) = u.pi; sd->alpha_set[j] = u.alpha; sd->omega_set[j] = u.omega;
        sd->zeta_set[j] = u.zeta; sd->beta_set[j] = be_j;
        const int slot = atomicAdd(&s_n, 1);
        sd->active[slot] = j;
        double *c = sd->coef + (size_t)slot * SH_COEF;
        c[0] = u.c1; c[1] = u.alpha; c[2] = u.c2; c[3] = u.c3; c[4] = be_j; c[5] = c4;
    }
    __syncthreads();
    if (t == 0) {
        sd->n_active = s_n;
        double max_zeta_pi = 1.0;                                                   // :451-476
        for (int j = 0; j < L; ++j) {
            if (sd->stop_flag[j]) continue;
            const double azp = (j == seed) ? 1.0 : fabs(1.0 / (sd->zeta_set[j] * PI(j, k)));
            if (azp * azp * sd->dot_r <= sd->tol * sd->tol * sd->dot_zero) {
                sd->stop_flag[j] = 1; sd->stop_count += 1; sd->stop_iter[j] = k;
            } else if (azp > max_zeta_pi) {
                max_zeta_pi = azp; sd->max_sigma = j;
            }
        }
    }
    __syncthreads();
    const bool sw = !sd->fixed && sd->stop_flag[seed] && sd->stop_count < L;        // :490 (shifted_lopbicg: never)
    if (sw) {
        const int ms = sd->max_sigma;
        const double dsg = sg_s - sd->sigma[ms];
        for (int i = 1 + t; i <= k; i += T) {                                       // :494-498
            const double ratio = PI(ms, i - 1) / PI(ms, i);
            sd->alpha_arch[i] = ratio * sd->alpha_arch[i];
            sd->beta_arch[i] = ratio * ratio * sd->beta_arch[i];
            sd->omega_arch[i] = sd->omega_arch[i] / (1.0 - sd->omega_arch[i] * dsg);
        }
        if (t == 0) sd->r_scale = 1.0 / (sd->zeta_set[ms] * PI(ms, k));            // :499
        __syncthreads();
        for (int j = t; j < L; j += T) { sd->eta_set[j] = 0.0; sd->zeta_set[j] = 1.0; }      // :501-505
        __syncthreads();
        const double sg_m = sd->sigma[ms];
        for (int j = t; j < L; j += T) {                                            // :509-517
            if (sd->stop_flag[j] || j == ms) continue;
            double eta = 0.0, zeta = 1.0;
            for (int i = 1; i <= k; ++i) {
                eta = (sd->beta_arch[i - 1] / sd->alpha_arch[i - 1]) * sd->alpha_arch[i] * eta - (sg_m - sd->sigma[j]) * sd->alpha_arch[i] * PI(j, i - 1);
                PI(j, i) = eta + PI(j, i - 1);
                zeta = (1.0 - sd->omega_arch[i] * (sg_m - sd->sigma[j])) * zeta;
            }
            sd->eta_set[j] = eta; sd->zeta_set[j] = zeta;
        }
        __syncthreads();
        if (sd->n_events < SH_EVENTS) {                                             // what the reference prints (:519-526)
            const int e = sd->n_events;
            for (int j = t; j < L; j += T) {
                double *v = sd->ev_vals + ((size_t)e * L + j) * 3;
                const bool shown = !(sd->stop_flag[j] || j == ms);
                v[0] = shown ? sd->eta_set[j] : NAN; v[1] = PI(j, k); v[2] = sd->zeta_set[j];
            }
        }
        __syncthreads();
        if (t == 0) {
            if (sd->n_events < SH_EVENTS) {
                sd->ev_k[sd->n_events] = k; sd->ev_seed[sd->n_events] = ms; sd->ev_remain[sd->n_events] = L - sd->stop_count;
                sd->n_events += 1;
            }
            sd->seed = ms; sd->sigma_seed = sd->sigma[ms]; sd->switched = 1;        // :524
        }
    }
    __syncthreads();
    if (t == 0) {
        sd->hist[k] = sd->dot_r / sd->dot_zero;
        sd->k = k + 1;                                                              // :537
        if (!(sd->stop_count < L && sd->k < sd->max_iter)) { sd->done = 1; sc->done = 1; }      // :372 (sc->done stops the shared kernels)
    }
}

// ---- vector kernels -----------------------------------------------------------------------------------------------
struct ShVec {
    KernelCommon kc;
    const ShiftDev *sd;
    double *r, *rh, *p, *s, *y, *qc, *rold;      // arena vectors (own parts)
    double *x_set, *p_set;
    long long stride;                            // doubles between consecutive shifts in both (even: every block starts 16-byte aligned)
    int n, L;
    int chunk;                                   // shifts per pass of sh_vec_shift, the size of its coefficient table (<= L)
};

// r# = r, p[seed] (arena) = r, p[j] = r for every shift, (r,r)                                        :342-354
__global__ void __launch_bounds__(256) sh_vec_init(const __grid_constant__ ShVec a)
{
    __shared__ double scratch[32 * MAX_DOTS];
    double dot[1] = {0.0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        const double r = a.r[i];
        a.rh[i] = r; a.p[i] = r;
        for (int j = 0; j < a.L; ++j) a.p_set[(size_t)j * a.stride + i] = r;
        dot[0] = fma(r, r, dot[0]);
    }
    block_sum<1>(dot, scratch);
    kernel_tail<1>(a.kc, dot, scratch);
}
// r_old = r; q = r - alpha s (in r); q_copy = q                                                       :374, 391-392
__global__ void __launch_bounds__(256) sh_vec_q(const __grid_constant__ ShVec a)
{
    if (a.sd->done) return;
    const double al = a.kc.sc->alpha;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        const double r = a.r[i];
        const double q = fma(-al, a.s[i], r);
        a.rold[i] = r; a.r[i] = q; a.qc[i] = q;
    }
}
// x[seed] += alpha p + omega q; r = q - omega y; (r,r), (r#,r)                                         :411-416
__global__ void __launch_bounds__(256) sh_vec_xr(const __grid_constant__ ShVec a)
{
    if (a.sd->done) return;
    __shared__ double scratch[32 * MAX_DOTS];
    const double al = a.kc.sc->alpha, om = a.kc.sc->omega;
    double *x = a.x_set + (size_t)a.sd->seed * a.stride;
    double dot[2] = {0.0, 0.0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        const double q = a.r[i];
        double xv = fma(al, a.p[i], x[i]);
        xv = fma(om, q, xv);
        const double r = fma(-om, a.y[i], q);
        x[i] = xv; a.r[i] = r;
        dot[0] = fma(r, r, dot[0]);
        dot[1] = fma(a.rh[i], r, dot[1]);
    }
    block_sum<2>(dot, scratch);
    kernel_tail<2>(a.kc, dot, scratch);
}
// all active shifts at once                                                                            :435-445
//   x_j += c1 q + alpha_j p_j ;  p_j += c2 q + c3 r_old ;  p_j = beta_j p_j + c4 r
// Two rows per thread, moved by the row-pair accesses of shifted_run.cuh.
// The active shifts go in passes of a.chunk: each pass loads their coefficients into shared memory and walks the rows.  A shift
// is updated in exactly one pass, with the same operations, so the number of passes does not change any result.
__global__ void __launch_bounds__(256) sh_vec_shift(const __grid_constant__ ShVec a)
{
    const ShiftDev *sd = a.sd;
    if (!sd->live) return;
    extern __shared__ double s_coef[];                       // [chunk][SH_COEF] then the shift indices
    int *s_idx = reinterpret_cast<int *>(s_coef + (size_t)a.chunk * SH_COEF);
    const int n_active = sd->n_active;
    for (int t0 = 0; t0 < n_active; t0 += a.chunk) {
        const int na = min(a.chunk, n_active - t0);
        __syncthreads();                                     // the previous pass is done with the table
        for (int t = threadIdx.x; t < na * SH_COEF; t += blockDim.x) s_coef[t] = sd->coef[(size_t)t0 * SH_COEF + t];
        for (int t = threadIdx.x; t < na; t += blockDim.x) s_idx[t] = sd->active[t0 + t];
        __syncthreads();
        for (int i = 2 * (blockIdx.x * blockDim.x + threadIdx.x); i < a.n; i += 2 * gridDim.x * blockDim.x) {
            const bool two = i + 1 < a.n;
            double q[2], o[2], r[2];
            ld2(a.qc, i, two, q); ld2(a.rold, i, two, o); ld2(a.r, i, two, r);
#pragma unroll 2
            for (int t = 0; t < na; ++t) {
                const double *c = s_coef + (size_t)t * SH_COEF;
                double *xj = a.x_set + (size_t)s_idx[t] * a.stride + i, *pj = a.p_set + (size_t)s_idx[t] * a.stride + i;
                double x[2], p[2];
                ld2(xj, 0, two, x); ld2(pj, 0, two, p);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    x[e] = fma(c[0], q[e], x[e]); x[e] = fma(c[1], p[e], x[e]);
                    p[e] = fma(c[2], q[e], p[e]); p[e] = fma(c[3], o[e], p[e]); p[e] = c[4] * p[e]; p[e] = fma(c[5], r[e], p[e]);
                }
                st2(xj, 0, two, x); st2(pj, 0, two, p);
            }
        }
    }
}
// The next SpMV input: normally p[seed] = r + beta p[seed] - beta omega s (:421-423, same operation order as solver.c:117-119);
// on a seed switch the old seed's p is dead, r <- r / (zeta pi) (:499) and the new seed's p (just advanced by sh_vec_shift)
// takes its place in the arena.
__global__ void __launch_bounds__(256) sh_vec_p(const __grid_constant__ ShVec a)
{
    const ShiftDev *sd = a.sd;
    if (!sd->live) return;
    if (sd->switched) {
        const double sc = sd->r_scale;
        const double *pn = a.p_set + (size_t)sd->seed * a.stride;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
            a.r[i] = sc * a.r[i];
            a.p[i] = pn[i];
        }
    } else {
        const double be = a.kc.sc->beta, nbo = -a.kc.sc->beta * a.kc.sc->omega;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
            double t = be * a.p[i];
            t = fma(1.0, a.r[i], t);
            a.p[i] = fma(nbo, a.s[i], t);
        }
    }
}

struct ShRun : PhaseLauncher {
    ShiftDev *d_sd = nullptr;
    ShVec base{};
    int ugrid = 1;                                   // grid of sh_vec_shift
    using PhaseLauncher::PhaseLauncher;

    ShVec vargs(TailDesc tail) const
    {
        ShVec v = base;
        v.kc = common(tail);
        return v;
    }
    void prologue()
    {
        sh_vec_init<<<m->vgrid, 256, 0, stream>>>(vargs(tail_store(1)));            // :342-354
        check_launch("sh_vec_init");
        sh_scalar_init<<<1, 256, 0, stream>>>(d_sd, m->d_sc);
        check_launch("sh_scalar_init");
        vec(PH_PUSH, tail_none(), V_P);
        c.launches += 2;
    }
    void iteration()
    {
        const int G = m->vgrid;
        const double *Y = nullptr;
        spmv(V_P, V_S, tail_store(1), 1, m->vec(V_RH), Y);                            // s = (A + sigma I) p, (r#,s)   :377-387
        sh_scalar_alpha<<<1, 1, 0, stream>>>(d_sd, m->d_sc);
        check_launch("sh_scalar_alpha");
        sh_vec_q<<<G, 256, 0, stream>>>(vargs(tail_none()));                          // q, r_old, q_copy            :374, 391-392
        check_launch("sh_vec_q");
        vec(PH_PUSH, tail_none(), V_R);
        spmv(V_R, V_Y, tail_store(2), 2, m->vec(V_R), m->vec(V_R), m->vec(V_R), Y);   // y = (A + sigma I) q, (q,q), (q,y)  :395-406
        sh_scalar_omega<<<1, 1, 0, stream>>>(d_sd, m->d_sc);
        check_launch("sh_scalar_omega");
        sh_vec_xr<<<G, 256, 0, stream>>>(vargs(tail_store(2)));                       // x[seed], r, (r,r), (r#,r)   :411-416
        check_launch("sh_vec_xr");
        sh_scalar_iter<<<1, 512, 0, stream>>>(d_sd, m->d_sc);                         // beta ... loop test          :420, 429-537
        check_launch("sh_scalar_iter");
        sh_vec_shift<<<ugrid, 256, (size_t)base.chunk * SH_ENTRY, stream>>>(vargs(tail_none()));     // x_j, p_j   :435-445
        check_launch("sh_vec_shift");
        sh_vec_p<<<G, 256, 0, stream>>>(vargs(tail_none()));                          // p[seed] (or the switch)     :421-423 / :499
        check_launch("sh_vec_p");
        vec(PH_PUSH, tail_none(), V_P);
        c.launches += 7;
    }
};

// The state of a new solve: the template (pointers, L) and the solve's own settings.  Every other field starts at zero, as the
// host struct it replaces did; sh_scalar_init sets the rest.
__global__ void sh_begin_kernel(ShiftDev *sd, const ShiftDev *tmpl, int fixed, int seed, double tol, int max_iter)
{
    *sd = *tmpl;
    sd->fixed = fixed; sd->seed = seed; sd->tol = tol; sd->max_iter = max_iter;
}

// what switching_solve reports (its return value, bicg_stats, bicg_last_shift_info), with the same IEEE operations
__global__ void sh_result_kernel(const ShiftDev *sd, const Scalars *sc, bicg_shift_result *out, int *stop_iter, ShiftHistRef *last)
{
    const int k = sd->k;
    if (threadIdx.x == 0) {
        last->hist = sd->hist; last->n = max(k, 1);
        if (out) {
            out->ret = sd->fixed ? k - 1 : k;
            out->iters = k - 1;
            out->converged = sd->stop_count >= sd->L;
            out->seed = sd->seed;
            out->error = sc->error;
            out->reserved = 0;
            out->final_res = sqrt(sd->dot_r / sd->dot_zero);
        }
    }
    if (stop_iter)
        for (int j = threadIdx.x; j < sd->L; j += blockDim.x) stop_iter[j] = sd->stop_iter[j];
}

// every device buffer of a solve with s.L shifts and max_iter (= SHIFT_MAX_ITER + 1) iterations, as the template of its state;
// p_set in *d_p
ShiftDev sh_buffers(ShiftedSolve &s, int max_iter, double **d_p)
{
    const int L = s.L;
    ShiftDev h{};
    h.L = L;
    h.sigma = s.alloc<double>(L);
    h.alpha_set = s.alloc<double>(L); h.beta_set = s.alloc<double>(L);
    h.omega_set = s.alloc<double>(L); h.eta_set = s.alloc<double>(L);
    h.zeta_set = s.alloc<double>(L);
    h.stop_flag = s.alloc<unsigned char>(L); h.stop_iter = s.alloc<int>(L);
    h.alpha_arch = s.alloc<double>(max_iter); h.beta_arch = s.alloc<double>(max_iter);
    h.omega_arch = s.alloc<double>(max_iter);
    h.pi_arch = s.alloc<double>((size_t)L * max_iter);
    h.coef = s.alloc<double>((size_t)L * SH_COEF); h.active = s.alloc<int>(L);
    h.hist = s.alloc<double>((size_t)max_iter + 1);
    h.ev_k = s.alloc<int>(SH_EVENTS); h.ev_seed = s.alloc<int>(SH_EVENTS);
    h.ev_remain = s.alloc<int>(SH_EVENTS);
    h.ev_vals = s.alloc<double>((size_t)SH_EVENTS * L * 3);
    *d_p = s.alloc<double>((size_t)L * s.stride);
    return h;
}

// the launcher of a solve on s's stream with state d_sd and p_set d_p
ShRun sh_run(ShiftedSolve &s, ShiftDev *d_sd, double *d_p)
{
    bicg_matrix *m = s.m;
    ShRun run(m, s.st);
    run.d_sd = d_sd;
    run.shift_sigma = &d_sd->sigma_seed;
    run.base.sd = d_sd;
    run.base.r = m->vec(V_R); run.base.rh = m->vec(V_RH); run.base.p = m->vec(V_P); run.base.s = m->vec(V_S);
    run.base.y = m->vec(V_Y); run.base.qc = m->vec(V_W); run.base.rold = m->vec(V_V);
    run.base.x_set = s.ws.d_x; run.base.p_set = d_p; run.base.stride = s.stride;
    run.base.n = s.n; run.base.L = s.L;
    run.ugrid = s.update_grid();
    run.base.chunk = std::min(s.L, table_chunk(sh_vec_shift, SH_ENTRY));
    return run;
}

// The enqueue half of every switching / fixed-seed solve on s.st, synchronous or asynchronous: the state from the workspace's
// template, the inputs (x_set and b moved by `in`, sigma by `sigma_in`), the reference's timed region (:364).  The outputs are
// s.finish / s.outputs.
void sh_enqueue(ShiftedSolve &s, const double *x_set, const double *r, const double *sigma, cudaMemcpyKind in, cudaMemcpyKind sigma_in,
                bool fixed, int seed)
{
    const Config &cfg = s.c.cfg;
    const int max_iter = cfg.shift_max_iter + 1;                                      // :293 (shifted_lopbicg: k from 0, :53-55)
    ShiftDev h;
    memcpy(&h, s.ws.tmpl.data(), sizeof(ShiftDev));
    ShiftDev *d_sd = (ShiftDev *)s.ws.d_state;
    BICG_CUDA(cudaMemsetAsync(h.pi_arch, 0, (size_t)s.L * max_iter * sizeof(double), s.st));
    BICG_CUDA(cudaMemsetAsync(h.hist, 0, ((size_t)max_iter + 1) * sizeof(double), s.st));
    s.upload(x_set, r, sigma, h.sigma, in, sigma_in);
    sh_begin_kernel<<<1, 1, 0, s.st>>>(d_sd, (const ShiftDev *)s.ws.d_tmpl, fixed ? 1 : 0, seed, cfg.shift_tol, max_iter);
    check_launch("sh_begin_kernel");
    ShRun run = sh_run(s, d_sd, s.ws.d_p);
    s.run(run, max_iter, &d_sd->done, 0);
}

} // namespace

int switching_solve(bicg_matrix *m, ShiftWork &ws, bool fixed, double *x_set, double *r, const double *sigma, int seed,
                    cudaMemcpyKind in, cudaMemcpyKind back)
{
    ShiftedSolve s(m, ws, ctx().stream);
    Context &c = s.c;
    const int L = s.L;
    s.synchronous(r, in);
    sh_enqueue(s, x_set, r, sigma, in, cudaMemcpyHostToDevice, fixed, seed);
    const ShiftDev out = s.finish(x_set, r, back, (const ShiftDev *)ws.d_state);
    // ---- results ------------------------------------------------------------------------------------------------------
    const int k = out.k;
    c.last_hist.assign((size_t)std::max(k, 1), 0.0);
    BICG_CUDA(cudaMemcpy(c.last_hist.data(), out.hist, (size_t)std::max(k, 1) * sizeof(double), cudaMemcpyDeviceToHost));
    c.last_shift_stop.assign((size_t)L, 0);
    BICG_CUDA(cudaMemcpy(c.last_shift_stop.data(), out.stop_iter, (size_t)L * sizeof(int), cudaMemcpyDeviceToHost));
    c.last_shift_seed = out.seed;
    bicg_stats st = s.stats();
    st.iters = k - 1; st.converged = out.stop_count >= L; st.final_res = sqrt(out.dot_r / out.dot_zero);
    c.last_stats = st;

    if (c.rank == 0 && !c.cfg.quiet && fixed) {
        // shifted_lopbicg prints the MEASURE_TIME lines only, its average over the iterations performed (:241-242)
        print_times(s.ms * 1e-3, k - 1);
    } else if (c.rank == 0 && !c.cfg.quiet) {
        // what the reference prints: the seed switches (:518-526), then the MEASURE_TIME lines (:557-561)
        std::vector<int> ek(SH_EVENTS), es(SH_EVENTS), er(SH_EVENTS);
        std::vector<double> ev((size_t)SH_EVENTS * L * 3);
        BICG_CUDA(cudaMemcpy(ek.data(), out.ev_k, SH_EVENTS * sizeof(int), cudaMemcpyDeviceToHost));
        BICG_CUDA(cudaMemcpy(es.data(), out.ev_seed, SH_EVENTS * sizeof(int), cudaMemcpyDeviceToHost));
        BICG_CUDA(cudaMemcpy(er.data(), out.ev_remain, SH_EVENTS * sizeof(int), cudaMemcpyDeviceToHost));
        BICG_CUDA(cudaMemcpy(ev.data(), out.ev_vals, ev.size() * sizeof(double), cudaMemcpyDeviceToHost));
        for (int e = 0; e < out.n_events && e < SH_EVENTS; ++e) {
            for (int j = 0; j < L; ++j) {
                const double *v = &ev[((size_t)e * L + j) * 3];
                if (!std::isnan(v[0])) printf("sigma[%d] eta: %f, pi: %f, zeta: %f\n", j, v[0], v[1], v[2]);
            }
            printf("k: %d, seed: %d, remain: %d\n", ek[(size_t)e], es[(size_t)e], er[(size_t)e]);
        }
        printf("Total iter   : %d\n", k - 1);
        print_times(s.ms * 1e-3, k);
    }
    s.report_error(sigma, out.seed);
    return fixed ? k - 1 : k;                                                         // :255 / :600
}

void switching_prepare(bicg_matrix *m, ShiftWork &ws)
{
    Context &c = ctx();
    ShiftedSolve s(m, ws, c.stream);
    if (ws.mem.empty()) {
        ws.d_x = s.alloc<double>((size_t)s.L * s.stride);
        ws.d_b = s.alloc<double>(s.n);
        const ShiftDev h = sh_buffers(s, ws.cap + 1, &ws.d_p);
        ShiftDev *d_sd = s.alloc<ShiftDev>(2);
        ws.d_state = d_sd; ws.d_tmpl = d_sd + 1;
        ws.tmpl.assign((const unsigned char *)&h, (const unsigned char *)&h + sizeof(ShiftDev));
        BICG_CUDA(cudaMemcpyAsync(ws.d_tmpl, &h, sizeof(ShiftDev), cudaMemcpyHostToDevice, c.stream));
    }
    if (!ws.exec[0]) {                              // the body is the same for both methods: `fixed` is a device flag
        ShiftDev *d_sd = (ShiftDev *)ws.d_state;
        ShRun run = sh_run(s, d_sd, ws.d_p);
        s.capture_loop(run, &d_sd->done, 0);
    }
}

void switching_solve_async(bicg_matrix *m, ShiftWork &ws, bool fixed, double *x_set, double *r, const double *sigma, int seed,
                           cudaStream_t st, bicg_shift_result *result, int *stop_iter)
{
    ShiftedSolve s(m, ws, st);
    sh_enqueue(s, x_set, r, sigma, cudaMemcpyDeviceToDevice, cudaMemcpyDeviceToDevice, fixed, seed);
    s.outputs(x_set, r, cudaMemcpyDeviceToDevice);
    sh_result_kernel<<<1, 256, 0, st>>>((const ShiftDev *)ws.d_state, m->d_sc, result, stop_iter, m->d_shift_last);
    check_launch("sh_result_kernel");
}

namespace {

// the workspace of a method's family (0: switching and fixed seed, 1: LOP and PIPE-LOP) and its variant of the captured loop
int shift_family(int method) { return method == BICG_SHIFTED_LOP || method == BICG_SHIFTED_PIPE_LOP ? 1 : 0; }
int shift_variant(int method) { return method == BICG_SHIFTED_PIPE_LOP ? 1 : 0; }

bool shift_method_known(int method)
{
    return method == BICG_SHIFTED_SWITCHING || method == BICG_SHIFTED_LOP || method == BICG_SHIFTED_PIPE_LOP ||
           method == BICG_SHIFTED_LOPBICG;
}

bool shift_async_prepared(const bicg_matrix *m, int method, int L)
{
    const ShiftWork &ws = m->shift_ws[shift_family(method)];
    return m->ev_last && m->d_loop && m->d_shift_last && ws.L == L && ws.cap >= ctx().cfg.shift_max_iter &&
           ws.exec[shift_variant(method)];
}

// frees a workspace's graphs; its buffers go back to the pool, or are kept until the handle is destroyed (retire: a captured
// graph may still use them)
void drop_work(bicg_matrix *m, ShiftWork &ws, bool retire)
{
    Context &c = ctx();
    for (int v = 0; v < 2; ++v) {
        if (ws.exec[v]) cudaGraphExecDestroy(ws.exec[v]);
        if (ws.iters[v]) cudaGraphDestroy(ws.iters[v]);
    }
    for (void *p : ws.mem) {
        if (retire) m->shift_retired.push_back(p);
        else c.dev_free(p);
    }
    ws = ShiftWork();
}

// The workspace of `method`'s family for L shifts and the current BICG_SHIFT_MAX_ITER with the method's loop captured, on the
// library's stream behind the handle's last work.  One for another L or a smaller bound is replaced.  Not collective.
ShiftWork &shift_work(bicg_matrix *m, int method, int L)
{
    Context &c = ctx();
    ShiftWork &ws = m->shift_ws[shift_family(method)];
    if (!ws.mem.empty() && (ws.L != L || ws.cap < c.cfg.shift_max_iter)) {
        // outgrown: nothing may still run on the old buffers when they return to the pool
        BICG_CUDA(cudaStreamSynchronize(c.stream));
        if (m->ev_last) BICG_CUDA(cudaEventSynchronize(m->ev_last));
        drop_work(m, ws, m->captured);
    }
    if (ws.mem.empty()) { ws.L = L; ws.cap = c.cfg.shift_max_iter; }
    if (shift_family(method) == 0) switching_prepare(m, ws);
    else lop_prepare(m, ws, method == BICG_SHIFTED_PIPE_LOP);
    return ws;
}

} // namespace

int shifted_solve(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int L, int seed, bool device_vectors)
{
    ctx().ensure();
    if (!shift_method_known(method) || L <= 0 || seed < 0 || seed >= L) return -1;
    wait_handle(m);
    ShiftWork &ws = shift_work(m, method, L);
    const cudaMemcpyKind in = device_vectors ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    const cudaMemcpyKind back = device_vectors ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    switch (method) {
    case BICG_SHIFTED_SWITCHING: return switching_solve(m, ws, false, x_set, r, sigma, seed, in, back);
    case BICG_SHIFTED_LOPBICG:   return switching_solve(m, ws, true, x_set, r, sigma, seed, in, back);
    case BICG_SHIFTED_LOP:       return lop_solve(m, ws, false, x_set, r, sigma, seed, in, back);
    default:                     return lop_solve(m, ws, true, x_set, r, sigma, seed, in, back);
    }
}

void drop_shift_work(bicg_matrix *m)
{
    Context &c = ctx();
    for (ShiftWork &ws : m->shift_ws) drop_work(m, ws, false);
    for (void *p : m->shift_retired) c.dev_free(p);
    m->shift_retired.clear();
    if (m->d_shift_last) c.dev_free(m->d_shift_last);
    m->d_shift_last = nullptr;
}

} // namespace bicg

extern "C" int bicg_shifted_solve_async_prepare(bicg_matrix *m, int method, int L)
{
    using namespace bicg;
    Context &c = ctx();
    // collective, as bicg_shifted_solve_dev: every rank's verdict, method and sigma_len
    if (!ranks_agree(!m || !shift_method_known(method) || L <= 0, {method, L})) return -1;
    c.ensure();
    // on the library's stream: the history record's and the template's initial values
    stream_ordered({m}, c.stream, false, [&] {
        if (!m->d_shift_last) {
            m->d_shift_last = (ShiftHistRef *)c.dev_alloc(sizeof(ShiftHistRef));
            BICG_CUDA(cudaMemsetAsync(m->d_shift_last, 0, sizeof(ShiftHistRef), c.stream));
        }
        shift_work(m, method, L);
    });
    return 0;
}

extern "C" int bicg_shifted_solve_async(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int L, int seed,
                                        void *stream, bicg_shift_result *result, int *stop_iter)
{
    using namespace bicg;
    ctx().ensure();
    if (!m || !x_set || !r || !sigma || !shift_method_known(method) || L <= 0 || seed < 0 || seed >= L) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    const bool captured = capturing(st);
    if (!shift_async_prepared(m, method, L)) {
        if (captured) return -2;
        if (bicg_shifted_solve_async_prepare(m, method, L) != 0) return -1;
    }
    if (captured) m->captured = true;
    ShiftWork &ws = m->shift_ws[shift_family(method)];
    stream_ordered({m}, st, captured, [&] {
        switch (method) {
        case BICG_SHIFTED_SWITCHING: switching_solve_async(m, ws, false, x_set, r, sigma, seed, st, result, stop_iter); break;
        case BICG_SHIFTED_LOPBICG:   switching_solve_async(m, ws, true, x_set, r, sigma, seed, st, result, stop_iter); break;
        case BICG_SHIFTED_LOP:       lop_solve_async(m, ws, false, x_set, r, sigma, seed, st, result, stop_iter); break;
        default:                     lop_solve_async(m, ws, true, x_set, r, sigma, seed, st, result, stop_iter); break;
        }
    });
    return 0;
}

extern "C" int bicg_matrix_shift_history(bicg_matrix *m, double *out, int cap)
{
    using namespace bicg;
    Context &c = ctx();
    c.ensure();
    if (!m) return -1;
    if (!m->d_shift_last) return 0;
    wait_handle(m);
    ShiftHistRef ref{};
    BICG_CUDA(cudaMemcpyAsync(&ref, m->d_shift_last, sizeof(ShiftHistRef), cudaMemcpyDeviceToHost, c.stream));
    BICG_CUDA(cudaStreamSynchronize(c.stream));
    if (out && cap > 0 && ref.n > 0) {
        BICG_CUDA(cudaMemcpyAsync(out, ref.hist, (size_t)std::min(ref.n, cap) * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
        BICG_CUDA(cudaStreamSynchronize(c.stream));
    }
    return ref.n;
}
