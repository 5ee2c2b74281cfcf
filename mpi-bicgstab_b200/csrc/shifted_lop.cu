// shifted_lop.cu -- the LOP shifted BiCGStab solvers of shifted_solver.h for (A + sigma_j I) x_j = b, j = 0 .. sigma_len - 1:
//   LOP      shifted_lopbicgstab (shifted_solver.c:182-354; _v2 :357-529 and _nooverlap :531-701 are the same arithmetic)
//   PIPE-LOP shifted_pipe_lopbicgstab (:703-895; _nooverlap :897-1085 is the same arithmetic), the pipelined seed recurrences
//            of pipe_bicgstab (s, z, w, v, t) with the same per-shift updates.
// The seed never changes and no shift stops on its own: every non-seed shift is advanced in every iteration until
// max_zeta_pi^2 dot_r <= tol^2 dot_zero (max_zeta_pi = max(1, max_j |1 / (zeta_j pi_j)|)) or MAX_ITER.
//
// Per iteration the seed runs on the arena vectors with the shifted SpMV epilogue (y = A x + sigma_seed x, PhaseLauncher),
// one scalar kernel derives every shift's coefficients (lop_scalar_shift, with shift_step of shifted_run.cuh), and ONE fused
// pass (lop_vec_update) updates the seed's x and residual together with x_j and p_j of every shift, each read and written
// exactly once (32 B per row and shift).  The reference scales p_j at the START of an iteration (p_j = beta_j p_j + r /
// (pi zeta), :264-269); that step is moved into the same pass, where r of the iteration start is r_old, so the pass does
//   p_j = beta_j p_j + c4 r_old ;  x_j += c1 q + alpha_j p_j ;  p_j += c2 q + c3 r_old
// with the reference's operands and operation order.  Iteration 1 starts from p_j = 0, beta_j = 0, c4 = 1: p_j = r exactly.
// Element-wise order = the reference's call order with gcc's FMA contraction (y += a x -> fma(a, x, y)).
// Pinned undefined behaviour: PIPE-LOP reads omega[seed] and s, z, v before writing them in its first iteration (:795-803);
// they start at 0 here, as with the oracle's zero-filling malloc (DESIGN.md section 1).
#include "engine.hpp"
#include "shifted_run.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace bicg {

namespace {

constexpr int LOP_COEF = 6;         // per non-seed shift: beta_j, c4, c1, alpha_j, c2, c3

struct LopDev {
    int L, max_iter, seed, k, done;
    double tol;
    double sigma_seed;                                  // read by the SpMV epilogue
    double rTr, rTr_old, dot_r, dot_zero, max_zeta_pi;
    double alpha, alpha_old, beta, omega;               // alpha_set[seed], alpha_old, beta_set[seed], omega_set[seed]
    double *sigma, *eta, *zeta, *pi_old, *pi_new;       // [L]
    double *coef;                                       // [L - 1][LOP_COEF]; slot t is shift t < seed ? t : t + 1
    double *hist;                                       // [max_iter + 1]
};

__device__ __forceinline__ bool loop_go(const LopDev *sd)                      // :259 / :793
{
    return sd->max_zeta_pi * sd->max_zeta_pi * sd->dot_r > sd->tol * sd->tol * sd->dot_zero && sd->k < sd->max_iter;
}

// ---- scalar kernels ------------------------------------------------------------------------------------------------
// (r,r) of b; LOP: alpha_set[seed] = 1 (:246); PIPE-LOP: alpha_old = 1, alpha is set by lop_scalar_pipe_init (:786-787)
__global__ void lop_scalar_init(LopDev *sd, Scalars *sc, int pipe)
{
    const int t = threadIdx.x;
    if (t == 0) {
        sd->rTr = sc->pend[0]; sd->dot_r = sd->rTr; sd->dot_zero = sd->rTr;   // :255-256 / :788-789
        sd->k = 0; sd->done = 0; sd->max_zeta_pi = 1.0;
        sd->alpha = 1.0; sd->alpha_old = 1.0; sd->beta = 0.0; sd->omega = 0.0;
        sd->hist[0] = 1.0;
        if (!pipe && !loop_go(sd)) { sd->done = 1; sc->done = 1; }
    }
    for (int j = t; j < sd->L; j += blockDim.x) { sd->eta[j] = 0.0; sd->zeta[j] = 1.0; sd->pi_old[j] = 1.0; sd->pi_new[j] = 1.0; }   // :243-251
}
__global__ void lop_scalar_pipe_init(LopDev *sd, Scalars *sc)                  // alpha = (r,r) / (r,w)   :787
{
    sd->alpha = sd->rTr / sc->pend[0];
    if (!loop_go(sd)) { sd->done = 1; sc->done = 1; }
}
__global__ void lop_scalar_alpha(LopDev *sd, Scalars *sc)                      // LOP :272-276
{
    if (sd->done) return;
    sd->alpha_old = sd->alpha;
    sd->alpha = sd->rTr / sc->pend[0];
}
// omega from the two pending dots, then every shift's coefficients and max |1/(zeta pi)|: one block
//   LOP :264-270, 283-289, 293, 296-304, 313-318;  PIPE-LOP :804-809, 817-825, 829, 832-840, 860-865
__global__ void __launch_bounds__(512) lop_scalar_shift(LopDev *sd, Scalars *sc)
{
    if (sd->done) return;
    __shared__ double s_max[512 / 32];
    const int t = threadIdx.x, T = blockDim.x;
    const double om = sc->pend[0] / sc->pend[1];                                // (q,q)/(q,y) resp. (q,y)/(y,y)
    const double al = sd->alpha, al_o = sd->alpha_old, be_o = sd->beta, sg_s = sd->sigma_seed;
    const int seed = sd->seed;
    double mx = 1.0;
    for (int s = t; s < sd->L - 1; s += T) {
        const int j = s < seed ? s : s + 1;
        const double pi_oo = sd->pi_old[j], pi_o = sd->pi_new[j], zeta_o = sd->zeta[j];
        // p_j is scaled at the start of this iteration, so with the previous iteration's beta, pi and zeta (:264-269 / :804-809)
        const double be_j = (pi_oo / pi_o) * (pi_oo / pi_o) * be_o;              // :266 / :806
        const double c4 = 1.0 / (pi_o * zeta_o);                                // :268 / :808
        const ShiftStep u = shift_step(al, al_o, be_o, om, sg_s - sd->sigma[j], sd->eta[j], pi_o, zeta_o);
        sd->eta[j] = u.eta; sd->pi_old[j] = pi_o; sd->pi_new[j] = u.pi; sd->zeta[j] = u.zeta;    // pi_old <- pi_new, :270 / :817
        double *c = sd->coef + (size_t)s * LOP_COEF;
        c[0] = be_j; c[1] = c4; c[2] = u.c1; c[3] = u.alpha; c[4] = u.c2; c[5] = u.c3;
        const double azp = fabs(1.0 / (u.zeta * u.pi));                         // :316 / :863
        if (azp > mx) mx = azp;
    }
    for (int o = 16; o > 0; o >>= 1) { const double v = __shfl_xor_sync(0xffffffffu, mx, o); if (v > mx) mx = v; }
    if ((t & 31) == 0) s_max[t >> 5] = mx;
    __syncthreads();
    if (t == 0) {
        for (int w = 1; w < (T + 31) / 32; ++w) if (s_max[w] > mx) mx = s_max[w];
        sd->max_zeta_pi = mx;
        sd->omega = om;
    }
}
// beta, the loop test and the history once the fused pass's dots are known
//   LOP      pend = (r,r), (r#,r)                               :306-312, 323
//   PIPE-LOP pend = (r,r), (r#,r), (r#,w), (r#,s), (r#,z)       :842-859, 867
__global__ void lop_scalar_end(LopDev *sd, Scalars *sc, int pipe)
{
    if (sd->done) return;
    sd->dot_r = sc->pend[0];
    sd->rTr_old = sd->rTr;
    sd->rTr = sc->pend[1];
    sd->beta = (sd->alpha / sd->omega) * (sd->rTr / sd->rTr_old);
    if (pipe) {
        const double rTw = sc->pend[2], rTs = sc->pend[3], rTz = sc->pend[4];
        sd->alpha_old = sd->alpha;
        sd->alpha = sd->rTr / (rTw + sd->beta * (rTs - sd->omega * rTz));
    }
    sd->k += 1;
    sd->hist[sd->k] = sd->dot_r / sd->dot_zero;
    if (!loop_go(sd)) { sd->done = 1; sc->done = 1; }
}

// ---- vector kernels -----------------------------------------------------------------------------------------------
struct LopVec {
    KernelCommon kc;
    const LopDev *sd;
    double *r, *rh, *p, *s, *y, *z, *w, *v, *t, *rold;  // arena vectors (own parts); y, z, w, v, t as the algorithm uses them
    double *x_set, *p_set;
    long long stride;                                   // doubles between consecutive shifts in both (even: 16-byte aligned blocks)
    int n, L;
    int chunk;                                          // non-seed shifts per pass of lop_vec_update, the size of its table
};

// r# = r, p[seed] = r, (r,r); PIPE-LOP also zeroes s, z, v (pinned, see the top)          :240-252 / :763, 772-782
__global__ void __launch_bounds__(256) lop_vec_init(const __grid_constant__ LopVec a, int pipe)
{
    __shared__ double scratch[32 * MAX_DOTS];
    double dot[1] = {0.0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        const double r = a.r[i];
        a.rh[i] = r; a.p[i] = r;
        if (pipe) { a.s[i] = 0.0; a.z[i] = 0.0; a.v[i] = 0.0; }
        dot[0] = fma(r, r, dot[0]);
    }
    block_sum<1>(dot, scratch);
    kernel_tail<1>(a.kc, dot, scratch);
}
// LOP: r_old = r; q = r - alpha s (in r)                                                   :271, 277
__global__ void __launch_bounds__(256) lop_vec_q(const __grid_constant__ LopVec a)
{
    if (a.sd->done) return;
    const double al = a.sd->alpha;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        const double r = a.r[i];
        a.rold[i] = r; a.r[i] = fma(-al, a.s[i], r);
    }
}
// LOP: p[seed] = r + beta p[seed] - beta omega s                                           :319-321
__global__ void __launch_bounds__(256) lop_vec_p(const __grid_constant__ LopVec a)
{
    if (a.sd->done) return;
    const double be = a.sd->beta, nbo = -a.sd->beta * a.sd->omega;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        double t = be * a.p[i];
        t = fma(1.0, a.r[i], t);
        a.p[i] = fma(nbo, a.s[i], t);
    }
}
// PIPE-LOP: p, s, z recurrences; r_old = r; q = r - alpha s (in r); y = w - alpha z (in w); (q,y), (y,y)      :795-803, 810-814
__global__ void __launch_bounds__(256) lop_vec_pipe1(const __grid_constant__ LopVec a)
{
    if (a.sd->done) return;
    __shared__ double scratch[32 * MAX_DOTS];
    const double al = a.sd->alpha, be = a.sd->beta, om = a.sd->omega;
    double dot[2] = {0.0, 0.0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        const double r = a.r[i], w = a.w[i], s0 = a.s[i], z0 = a.z[i];
        double u = fma(-om, s0, a.p[i]);   u = be * u;  a.p[i] = fma(1.0, r, u);
        double sv = fma(-om, z0, s0);      sv = be * sv; sv = fma(1.0, w, sv);
        double zv = fma(-om, a.v[i], z0);  zv = be * zv; zv = fma(1.0, a.t[i], zv);
        const double q = fma(-al, sv, r), y = fma(-al, zv, w);
        a.s[i] = sv; a.z[i] = zv; a.rold[i] = r; a.r[i] = q; a.w[i] = y;
        dot[0] = fma(q, y, dot[0]);
        dot[1] = fma(y, y, dot[1]);
    }
    block_sum<2>(dot, scratch);
    kernel_tail<2>(a.kc, dot, scratch);
}
// The seed's x and residual and every shift's x_j, p_j in one pass over the rows (two rows per thread, moved by the row-pair
// accesses of shifted_run.cuh).
//   seed   x[seed] += alpha p + omega q; r = q - omega y                                   :294-295, 305 / :830-831, 841
//          PIPE-LOP: w = y - omega (t - alpha v)                                          :843-844
//   shifts p_j = beta_j p_j + c4 r_old; x_j += c1 q + alpha_j p_j; p_j += c2 q + c3 r_old   :267-268, 299-302 / :807-808, 835-838
//   dots   LOP (r,r), (r#,r)                                                               :306, 308
//          PIPE-LOP (r,r), (r#,r), (r#,w), (r#,s), (r#,z)                                  :842, 846-849
// The non-seed shifts go in passes of a.chunk, each of which loads their coefficients into shared memory and walks the rows;
// the seed is updated in the last pass, because that overwrites q (in r), which every earlier pass reads.  A shift is updated
// in exactly one pass, with the same operations, so the number of passes does not change any result.
template <bool PIPE, bool SEED>
__device__ __forceinline__ void lop_rows(const LopVec &a, const double *s_coef, int t0, int na, double (&dot)[PIPE ? 5 : 2])
{
    const LopDev *sd = a.sd;
    const int seed = sd->seed;
    const double al = sd->alpha, om = sd->omega;
    double *xs = a.x_set + (size_t)seed * a.stride;
    for (int i = 2 * (blockIdx.x * blockDim.x + threadIdx.x); i < a.n; i += 2 * gridDim.x * blockDim.x) {
        const bool two = i + 1 < a.n;                   // stride and arena vectors are 16-byte aligned, i is even
        double q[2], o[2];
        ld2(a.r, i, two, q); ld2(a.rold, i, two, o);
        if constexpr (SEED) {
            const int ne = two ? 2 : 1;
            double y[2], r[2], rh[2];
            ld2(a.rh, i, two, rh); ld2(PIPE ? a.w : a.y, i, two, y);
            for (int e = 0; e < ne; ++e) {
                r[e] = fma(-om, y[e], q[e]);
                dot[0] = fma(r[e], r[e], dot[0]);
                dot[1] = fma(rh[e], r[e], dot[1]);
            }
            st2(a.r, i, two, r);
            if constexpr (PIPE) {
                double t[2], v[2], w[2], s[2], z[2];
                ld2(a.t, i, two, t); ld2(a.v, i, two, v); ld2(a.s, i, two, s); ld2(a.z, i, two, z);
                for (int e = 0; e < ne; ++e) {
                    t[e] = fma(-al, v[e], t[e]);        // t itself is overwritten by t = (A + sigma I) w next
                    w[e] = fma(-om, t[e], y[e]);
                    dot[2] = fma(rh[e], w[e], dot[2]);
                    dot[3] = fma(rh[e], s[e], dot[3]);
                    dot[4] = fma(rh[e], z[e], dot[4]);
                }
                st2(a.w, i, two, w);
            }
            double x[2], p[2];                          // last: fewer values live at once (64 registers with PIPE)
            ld2(xs, i, two, x); ld2(a.p, i, two, p);
            for (int e = 0; e < ne; ++e) {
                x[e] = fma(al, p[e], x[e]);
                x[e] = fma(om, q[e], x[e]);
            }
            st2(xs, i, two, x);
        }
        if (!two) { q[1] = 0.0; o[1] = 0.0; }
#pragma unroll 2
        for (int t = 0; t < na; ++t) {
            const double *c = s_coef + (size_t)t * LOP_COEF;
            const size_t j = (size_t)(t0 + t < seed ? t0 + t : t0 + t + 1);
            double *xj = a.x_set + j * a.stride + i, *pj = a.p_set + j * a.stride + i;
            double xv[2], pv[2];
            ld2(xj, 0, two, xv); ld2(pj, 0, two, pv);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                pv[e] = c[0] * pv[e]; pv[e] = fma(c[1], o[e], pv[e]);
                xv[e] = fma(c[2], q[e], xv[e]); xv[e] = fma(c[3], pv[e], xv[e]);
                pv[e] = fma(c[4], q[e], pv[e]); pv[e] = fma(c[5], o[e], pv[e]);
            }
            st2(xj, 0, two, xv); st2(pj, 0, two, pv);
        }
    }
}
template <bool PIPE>
__global__ void __launch_bounds__(256) lop_vec_update(const __grid_constant__ LopVec a)
{
    const LopDev *sd = a.sd;
    if (sd->done) return;
    constexpr int ND = PIPE ? 5 : 2;
    __shared__ double scratch[32 * MAX_DOTS];
    extern __shared__ double s_coef[];                  // [chunk][LOP_COEF]
    const int n_shift = a.L - 1;
    double dot[ND];
#pragma unroll
    for (int d = 0; d < ND; ++d) dot[d] = 0.0;
    for (int t0 = 0;; t0 += a.chunk) {
        const int na = min(a.chunk, n_shift - t0);
        __syncthreads();                                // the previous pass is done with the table
        for (int t = threadIdx.x; t < na * LOP_COEF; t += blockDim.x) s_coef[t] = sd->coef[(size_t)t0 * LOP_COEF + t];
        __syncthreads();
        if (t0 + na >= n_shift) {
            lop_rows<PIPE, true>(a, s_coef, t0, na, dot);
            break;
        }
        lop_rows<PIPE, false>(a, s_coef, t0, na, dot);
    }
    block_sum<ND>(dot, scratch);
    kernel_tail<ND>(a.kc, dot, scratch);
}

struct LopRun : PhaseLauncher {
    LopDev *d_sd = nullptr;
    LopVec base{};
    bool pipe = false;
    int ugrid = 1;                                      // grid of lop_vec_update
    using PhaseLauncher::PhaseLauncher;

    LopVec vargs(TailDesc tail) const
    {
        LopVec v = base;
        v.kc = common(tail);
        return v;
    }
    void prologue()
    {
        const int G = m->vgrid;
        lop_vec_init<<<G, 256, 0, stream>>>(vargs(tail_store(1)), pipe ? 1 : 0);
        check_launch("lop_vec_init");
        lop_scalar_init<<<1, 256, 0, stream>>>(d_sd, m->d_sc, pipe ? 1 : 0);
        check_launch("lop_scalar_init");
        c.launches += 2;
        if (!pipe) { vec(PH_PUSH, tail_none(), V_P); return; }
        vec(PH_PUSH, tail_none(), V_R);
        spmv(V_R, V_W, tail_store(1), 1, m->vec(V_R), nullptr);                         // w = (A + sigma I) r, (r,w)  :765-767
        lop_scalar_pipe_init<<<1, 1, 0, stream>>>(d_sd, m->d_sc);                      // alpha                       :787
        check_launch("lop_scalar_pipe_init");
        vec(PH_PUSH, tail_none(), V_W);
        spmv(V_W, V_T, tail_none());                                                   // t = (A + sigma I) w          :769-770
        c.launches += 1;
    }
    void iteration()
    {
        const int G = m->vgrid;
        const size_t smem = (size_t)base.chunk * LOP_COEF * sizeof(double);
        if (!pipe) {
            spmv(V_P, V_S, tail_store(1), 1, m->vec(V_RH), nullptr);                    // s = (A + sigma I) p, (r#,s)   :261-263
            lop_scalar_alpha<<<1, 1, 0, stream>>>(d_sd, m->d_sc);                      // alpha                        :276
            check_launch("lop_scalar_alpha");
            lop_vec_q<<<G, 256, 0, stream>>>(vargs(tail_none()));                      // r_old, q                     :271, 277
            check_launch("lop_vec_q");
            vec(PH_PUSH, tail_none(), V_R);
            spmv(V_R, V_Y, tail_store(2), 2, m->vec(V_R), m->vec(V_R), m->vec(V_R), nullptr);   // y = (A + sigma I) q, (q,q), (q,y)  :278-282
            lop_scalar_shift<<<1, 512, 0, stream>>>(d_sd, m->d_sc);                    // omega, every shift's scalars
            check_launch("lop_scalar_shift");
            lop_vec_update<false><<<ugrid, 256, smem, stream>>>(vargs(tail_store(2)));
            check_launch("lop_vec_update");
            lop_scalar_end<<<1, 1, 0, stream>>>(d_sd, m->d_sc, 0);                     // beta, loop test              :312-318
            check_launch("lop_scalar_end");
            lop_vec_p<<<G, 256, 0, stream>>>(vargs(tail_none()));                      // p[seed]                      :319-321
            check_launch("lop_vec_p");
            vec(PH_PUSH, tail_none(), V_P);
            c.launches += 6;
        } else {
            lop_vec_pipe1<<<G, 256, 0, stream>>>(vargs(tail_store(2)));                // p, s, z, q, y, (q,y), (y,y)   :795-814
            check_launch("lop_vec_pipe1");
            vec(PH_PUSH, tail_none(), V_Z);
            spmv(V_Z, V_V, tail_none());                                               // v = (A + sigma I) z           :815-816
            lop_scalar_shift<<<1, 512, 0, stream>>>(d_sd, m->d_sc);                    // omega, every shift's scalars
            check_launch("lop_scalar_shift");
            lop_vec_update<true><<<ugrid, 256, smem, stream>>>(vargs(tail_store(5)));
            check_launch("lop_vec_update");
            vec(PH_PUSH, tail_none(), V_W);
            spmv(V_W, V_T, tail_none());                                               // t = (A + sigma I) w           :850-851
            lop_scalar_end<<<1, 1, 0, stream>>>(d_sd, m->d_sc, 1);                     // beta, alpha, loop test       :857-865
            check_launch("lop_scalar_end");
            c.launches += 4;
        }
    }
};

// The state of a new solve: the template (pointers, L) and the solve's own settings, sigma_seed from the staged sigma (read by the
// SpMV epilogue from the first kernel on).  Every other field starts at zero; lop_scalar_init sets the rest.
__global__ void lop_begin_kernel(LopDev *sd, const LopDev *tmpl, int seed, double tol, int max_iter)
{
    *sd = *tmpl;
    sd->seed = seed; sd->tol = tol; sd->max_iter = max_iter;
    sd->sigma_seed = sd->sigma[seed];
}

// what lop_solve reports (its return value, bicg_stats, bicg_last_shift_info), with the same IEEE operations
__global__ void lop_result_kernel(const LopDev *sd, const Scalars *sc, bicg_shift_result *out, int *stop_iter, ShiftHistRef *last)
{
    const int k = sd->k;
    if (threadIdx.x == 0) {
        last->hist = sd->hist; last->n = k + 1;
        if (out) {
            out->ret = k;
            out->iters = k;
            out->converged = sd->max_zeta_pi * sd->max_zeta_pi * sd->dot_r <= sd->tol * sd->tol * sd->dot_zero;
            out->seed = sd->seed;
            out->error = sc->error;
            out->reserved = 0;
            out->final_res = sqrt(sd->dot_r / sd->dot_zero);
        }
    }
    if (stop_iter)                                      // no shift stops on its own
        for (int j = threadIdx.x; j < sd->L; j += blockDim.x) stop_iter[j] = 0;
}

// every device buffer of a solve with s.L shifts and max_iter iterations, as the template of its state; p_set in *d_p
LopDev lop_buffers(ShiftedSolve &s, int max_iter, double **d_p)
{
    const int L = s.L;
    LopDev h{};
    h.L = L;
    h.sigma = s.alloc<double>(L);
    h.eta = s.alloc<double>(L); h.zeta = s.alloc<double>(L);
    h.pi_old = s.alloc<double>(L); h.pi_new = s.alloc<double>(L);
    h.coef = s.alloc<double>((size_t)(L - 1) * LOP_COEF);
    h.hist = s.alloc<double>((size_t)max_iter + 1);
    *d_p = s.alloc<double>((size_t)L * s.stride);
    return h;
}

// the launcher of a solve on s's stream with state d_sd and p_set d_p
LopRun lop_run(ShiftedSolve &s, bool pipe, LopDev *d_sd, double *d_p)
{
    bicg_matrix *m = s.m;
    LopRun run(m, s.st);
    run.pipe = pipe;
    run.d_sd = d_sd;
    run.shift_sigma = &d_sd->sigma_seed;
    run.base.sd = d_sd;
    run.base.r = m->vec(V_R); run.base.rh = m->vec(V_RH); run.base.p = m->vec(V_P); run.base.s = m->vec(V_S);
    run.base.y = m->vec(V_Y); run.base.z = m->vec(V_Z); run.base.w = m->vec(V_W); run.base.v = m->vec(V_V); run.base.t = m->vec(V_T);
    run.base.rold = m->vec(pipe ? V_AX : V_V);
    run.base.x_set = s.ws.d_x; run.base.p_set = d_p; run.base.stride = s.stride;
    run.base.n = s.n; run.base.L = s.L;
    run.ugrid = s.update_grid();
    constexpr size_t entry = LOP_COEF * sizeof(double);
    run.base.chunk = std::min(s.L - 1, pipe ? table_chunk(lop_vec_update<true>, entry) : table_chunk(lop_vec_update<false>, entry));
    return run;
}

// The enqueue half of every LOP / PIPE-LOP solve on s.st, synchronous or asynchronous: the state from the workspace's template,
// the inputs (x_set and b moved by `in`, sigma by `sigma_in`), the reference's timed region (:237 / :759).  The outputs are
// s.finish / s.outputs.
void lop_enqueue(ShiftedSolve &s, bool pipe, const double *x_set, const double *r, const double *sigma, cudaMemcpyKind in,
                 cudaMemcpyKind sigma_in, int seed)
{
    const Config &cfg = s.c.cfg;
    const int max_iter = cfg.shift_max_iter;
    LopDev h;
    memcpy(&h, s.ws.tmpl.data(), sizeof(LopDev));
    LopDev *d_sd = (LopDev *)s.ws.d_state;
    BICG_CUDA(cudaMemsetAsync(h.hist, 0, ((size_t)max_iter + 1) * sizeof(double), s.st));
    BICG_CUDA(cudaMemsetAsync(s.ws.d_p, 0, (size_t)s.L * s.stride * sizeof(double), s.st));   // p_loc_set = calloc(...)  :226
    s.upload(x_set, r, sigma, h.sigma, in, sigma_in);
    lop_begin_kernel<<<1, 1, 0, s.st>>>(d_sd, (const LopDev *)s.ws.d_tmpl, seed, cfg.shift_tol, max_iter);
    check_launch("lop_begin_kernel");
    LopRun run = lop_run(s, pipe, d_sd, s.ws.d_p);
    s.run(run, max_iter, &d_sd->done, pipe ? 1 : 0);
}

} // namespace

int lop_solve(bicg_matrix *m, ShiftWork &ws, bool pipe, double *x_set, double *r, const double *sigma, int seed, cudaMemcpyKind in,
              cudaMemcpyKind back)
{
    ShiftedSolve s(m, ws, ctx().stream);
    Context &c = s.c;
    const int L = s.L;
    s.synchronous(r, in);
    lop_enqueue(s, pipe, x_set, r, sigma, in, cudaMemcpyHostToDevice, seed);
    const LopDev out = s.finish(x_set, r, back, (const LopDev *)ws.d_state);

    // ---- results ------------------------------------------------------------------------------------------------------
    const int k = out.k;
    c.last_hist.assign((size_t)k + 1, 0.0);
    BICG_CUDA(cudaMemcpy(c.last_hist.data(), out.hist, ((size_t)k + 1) * sizeof(double), cudaMemcpyDeviceToHost));
    bicg_stats st = s.stats();
    const double res = sqrt(out.dot_r / out.dot_zero);
    st.iters = k;
    st.converged = out.max_zeta_pi * out.max_zeta_pi * out.dot_r <= out.tol * out.tol * out.dot_zero;      // false after a NaN
    st.final_res = res;
    c.last_stats = st;
    c.last_shift_stop.assign((size_t)L, 0);                                           // no shift stops on its own
    c.last_shift_seed = seed;

    if (c.rank == 0 && !c.cfg.quiet) {                                                // :339-346 / :882-889
        printf("Total iter   : %d\n", k);
        printf("Final r      : %e\n", res);
        print_times(s.ms * 1e-3, k);
    }
    s.report_error(sigma, seed);
    return k;                                                                         // :352 / :894
}

void lop_prepare(bicg_matrix *m, ShiftWork &ws, bool pipe)
{
    Context &c = ctx();
    ShiftedSolve s(m, ws, c.stream);
    if (ws.mem.empty()) {
        ws.d_x = s.alloc<double>((size_t)s.L * s.stride);
        ws.d_b = s.alloc<double>(s.n);
        const LopDev h = lop_buffers(s, ws.cap, &ws.d_p);
        LopDev *d_sd = s.alloc<LopDev>(2);
        ws.d_state = d_sd; ws.d_tmpl = d_sd + 1;
        ws.tmpl.assign((const unsigned char *)&h, (const unsigned char *)&h + sizeof(LopDev));
        BICG_CUDA(cudaMemcpyAsync(ws.d_tmpl, &h, sizeof(LopDev), cudaMemcpyHostToDevice, c.stream));
    }
    const int v = pipe ? 1 : 0;
    if (!ws.exec[v]) {
        LopDev *d_sd = (LopDev *)ws.d_state;
        LopRun run = lop_run(s, pipe, d_sd, ws.d_p);
        s.capture_loop(run, &d_sd->done, v);
    }
}

void lop_solve_async(bicg_matrix *m, ShiftWork &ws, bool pipe, double *x_set, double *r, const double *sigma, int seed,
                     cudaStream_t st, bicg_shift_result *result, int *stop_iter)
{
    ShiftedSolve s(m, ws, st);
    lop_enqueue(s, pipe, x_set, r, sigma, cudaMemcpyDeviceToDevice, cudaMemcpyDeviceToDevice, seed);
    s.outputs(x_set, r, cudaMemcpyDeviceToDevice);
    lop_result_kernel<<<1, 256, 0, st>>>((const LopDev *)ws.d_state, m->d_sc, result, stop_iter, m->d_shift_last);
    check_launch("lop_result_kernel");
}

} // namespace bicg
