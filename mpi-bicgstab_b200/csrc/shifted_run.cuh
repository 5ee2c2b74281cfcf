// shifted_run.cuh -- host-side launch helpers shared by the shifted solvers (shifted.cu, shifted_lop.cu): the halo push of an
// arena vector before an SpMV (kernel-per-phase protocol) and the SpMV y = (A + sigma_seed I) x with up to two epilogue dots
// whose totals land in Scalars::pend[] for the solver's own scalar kernels.
#pragma once
#include "engine.hpp"

namespace bicg {
namespace {

inline TailDesc tail_none() { return TailDesc{TAIL_NONE, FIN_NONE, 0, 0, 0, 0, 0}; }
inline TailDesc tail_store(int ndot) { return TailDesc{TAIL_ALLREDUCE, FIN_STORE_PEND, ndot, 0, 0, 0, 0}; }

__global__ void sh_reset_scalars(Scalars *s)
{
    s->alpha = s->beta = s->omega = 0.0;
    for (int k = 0; k < MAX_DOTS; ++k) s->pend[k] = 0.0;
    s->k = 0; s->max_iter = 0; s->done = 0; s->converged = 0; s->error = 0; s->ticket = 0u;
}

struct ShiftLaunch {
    bicg_matrix *m;
    Context &c;
    const double *shift_sigma = nullptr;          // device scalar the SpMV epilogue adds as sigma x
    int launches = 0;
    explicit ShiftLaunch(bicg_matrix *mm) : m(mm), c(ctx()) {}

    PushDesc make_push(int id) const
    {
        PushDesc pd{};
        if (m->world == 1) return pd;
        pd.npeers = m->npush; pd.fence_writers = c.cfg.fence_writers;
        pd.src = m->vec(id);
        for (int s = 0; s < m->npush; ++s) {
            const int d = m->push_peer[s];
            pd.dst[s] = (double *)((char *)m->peer_base[d] + m->peer_vec_off[d]) + (long long)id * m->peer_vstride[d] + m->peer_ghost_off[d];
            pd.runs[s] = m->d_push_runs[s]; pd.nruns[s] = m->push_nruns[s];
        }
        return pd;
    }
    VecArgs vec_args(TailDesc tail) const
    {
        VecArgs a{};
        a.kc.sc = m->d_sc; a.kc.partials = m->d_partials; a.kc.hist = m->d_hist; a.kc.comm = m->comm; a.kc.tail = tail;
        a.v.x = m->vec(V_X); a.v.r = m->vec(V_R); a.v.rh = m->vec(V_RH); a.v.p = m->vec(V_P); a.v.s = m->vec(V_S);
        a.v.y = m->vec(V_Y); a.v.z = m->vec(V_Z); a.v.w = m->vec(V_W); a.v.v = m->vec(V_V); a.v.t = m->vec(V_T);
        a.v.b = m->vec(V_B); a.v.ax = m->vec(V_AX);
        a.n = m->n_loc; a.chunk = m->vchunk;
        return a;
    }
    void push(int id)                             // halo of arena vector `id` for the next SpMV (kernel-per-phase protocol)
    {
        if (m->world == 1) return;
        VecArgs a = vec_args(tail_none());
        a.kc.tail.signal_halo = 1;
        a.push = make_push(id);
        int rc = launch_vec(PH_PUSH, m->vgrid, a, c.stream);
        if (rc) fatal("bicgstab_b200: push kernel launch failed: %s", cudaGetErrorString((cudaError_t)rc));
        ++launches; ++c.launches;
    }
    // y = (A + sigma I) x; ndot (0..2) epilogue dots, a null b = the y just computed
    void spmv(int x_id, int y_id, int ndot, const double *a0 = nullptr, const double *b0 = nullptr, const double *a1 = nullptr,
              const double *b1 = nullptr)
    {
        SpmvArgs a = make_spmv_args(m, m->plan, x_id, y_id);
        a.kc.tail = ndot > 0 ? tail_store(ndot) : tail_none();
        a.shift_sigma = shift_sigma;
        if (ndot > 0) epi_add_dot(a.epi, a0, b0);
        if (ndot > 1) epi_add_dot(a.epi, a1, b1);
        launch_spmv_plan(m, m->plan, a, 0);
        ++launches;
    }
};

} // namespace
} // namespace bicg
