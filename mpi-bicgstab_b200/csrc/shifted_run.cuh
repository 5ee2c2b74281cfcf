// shifted_run.cuh -- what every shifted solver shares (shifted.cu, shifted_lop.cu).
// Host: the seed system runs on the arena vectors through PhaseLauncher (engine.hpp) with shift_sigma set, so its SpMVs
// compute y = (A + sigma_seed I) x, and tail_store puts the reduced epilogue dots into Scalars::pend[] for the solver's own
// scalar kernels.  ShiftedSolve holds everything around a solver's own device state and kernel sequence: the handle's workspace
// of the family (ShiftWork) with every buffer of the solve, the sigma_len solutions x_j staged in one strided device buffer,
// b in / the seed residual out through the arena's r, the update kernels' grid, the loop as a WHILE node and the statistics
// every synchronous shifted solver reports alike.  The synchronous and asynchronous solves run the same enqueue half and
// differ only in their stream, their copy kinds and their finish.
// Device: the per-shift scalar recurrence both families evaluate (shift_step) and the row-pair accesses their update
// kernels move x_j and p_j with (ld2, st2).  Each family keeps its own update loop: they apply the six
// coefficients in different orders, and LOP folds the seed's update into its last pass.
#pragma once
#include "engine.hpp"

#include <algorithm>
#include <vector>

namespace bicg {

// Each family (shifted.cu: fixed = shifted_lopbicg, else shifted_lopbicg_switching; shifted_lop.cu: pipe = PIPE-LOP, else LOP)
// has a prepare, which allocates workspace ws for ws.L shifts and ws.cap iterations when it is empty and captures the variant's
// loop when it has not been, and two enqueues with ws's buffers: *_solve, the synchronous solve on the library's stream
// (x_set and r moved by in / out, sigma a host array), and *_solve_async on st (x_set, r, sigma: device pointers; result,
// stop_iter: optional device outputs).  Both run with BICG_SHIFT_TOL and BICG_SHIFT_MAX_ITER.
void switching_prepare(bicg_matrix *m, ShiftWork &ws);
int  switching_solve(bicg_matrix *m, ShiftWork &ws, bool fixed, double *x_set, double *r, const double *sigma, int seed,
                     cudaMemcpyKind in, cudaMemcpyKind out);
void switching_solve_async(bicg_matrix *m, ShiftWork &ws, bool fixed, double *x_set, double *r, const double *sigma, int seed,
                           cudaStream_t st, bicg_shift_result *result, int *stop_iter);
void lop_prepare(bicg_matrix *m, ShiftWork &ws, bool pipe);
int  lop_solve(bicg_matrix *m, ShiftWork &ws, bool pipe, double *x_set, double *r, const double *sigma, int seed, cudaMemcpyKind in,
               cudaMemcpyKind out);
void lop_solve_async(bicg_matrix *m, ShiftWork &ws, bool pipe, double *x_set, double *r, const double *sigma, int seed,
                     cudaStream_t st, bicg_shift_result *result, int *stop_iter);

// After each launch of a shifted solver's own kernels: a launch that fails (its configuration, its shared memory) is reported
// at that kernel instead of at the next checked launch.
inline void check_launch(const char *kernel)
{
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) fatal("bicgstab_b200: %s launch failed: %s", kernel, cudaGetErrorString(e));
}
// Shifts per pass of an update kernel whose coefficient table in dynamic shared memory takes `entry` bytes per shift: as many
// as fit, next to the kernel's static shared memory, into the 48 KB a block gets without opting in to more.  The kernel walks
// its rows once per pass, so any number of shifts works with one launch configuration.
template <class Kernel> int table_chunk(Kernel kernel, size_t entry)
{
    cudaFuncAttributes fa{};
    BICG_CUDA(cudaFuncGetAttributes(&fa, kernel));
    return std::max(1, (int)((48 * 1024 - fa.sharedSizeBytes) / entry));
}

// One step of shift j's scalars from the seed's alpha_k, alpha_{k-1}, beta_{k-1}, omega_k, dsg = sigma_seed - sigma_j and
// the shift's eta, pi, zeta (shifted_switching_solver.c:431-441; shifted_solver.c:285-303 / :821-839).  beta_j and c4 stay
// with the callers, who take them one iteration apart.
struct ShiftStep {
    double eta, pi, alpha, omega, c1, c2, c3, zeta;     // eta, pi_new, alpha_j, omega_j, the update coefficients, zeta_new
};
__device__ __forceinline__ ShiftStep shift_step(double al, double al_o, double be_o, double om, double dsg, double eta, double pi_o,
                                                double zeta_o)
{
    ShiftStep s;
    s.eta = (be_o / al_o) * al * eta - dsg * al * pi_o;
    s.pi = s.eta + pi_o;
    s.alpha = (pi_o / s.pi) * al;
    s.omega = om / (1.0 - om * dsg);
    s.c1 = s.omega / (s.pi * zeta_o);
    s.c2 = s.omega / (s.alpha * zeta_o * s.pi);
    s.c3 = -s.omega / (s.alpha * zeta_o * pi_o);
    s.zeta = (1.0 - om * dsg) * zeta_o;
    return s;
}

// Rows i, i + 1 (two) or i alone of a vector, as one 16-byte access: the arena vectors and every x_set and p_set block start
// 16-byte aligned, and the update kernels give each thread an even i.
__device__ __forceinline__ void ld2(const double *p, int i, bool two, double (&v)[2])
{
    if (two) { const double2 t = *reinterpret_cast<const double2 *>(p + i); v[0] = t.x; v[1] = t.y; }
    else { v[0] = p[i]; v[1] = 0.0; }
}
__device__ __forceinline__ void st2(double *p, int i, bool two, const double (&v)[2])
{
    if (two) *reinterpret_cast<double2 *>(p + i) = make_double2(v[0], v[1]);
    else p[i] = v[0];
}

struct ShiftedSolve {
    static constexpr int U = 8;              // iterations per body of the device-side loop
    bicg_matrix *m;
    Context &c;
    ShiftWork &ws;                           // the handle's workspace of the family: every buffer, x_set staged in ws.d_x
    const int n, L;
    const cudaStream_t st;                   // where the solve is enqueued: the library's stream, or the caller's
    const long long stride;                  // doubles between consecutive shifts in d_x and p_set (16-byte aligned blocks)
    float ms = 0.f;                          // synchronous solve: length of the timed region
    int launches0 = 0, bodies = 0, variant = 0;
    uint64_t pcie_bytes = 0;                 // ... x_set and b in / x_set and r out, each way, when they are host arrays

    ShiftedSolve(bicg_matrix *mm, ShiftWork &w, cudaStream_t s)
        : m(mm), c(ctx()), ws(w), n(mm->n_loc), L(w.L), st(s), stride(((long long)mm->n_loc + 15) / 16 * 16) {}
    ShiftedSolve(const ShiftedSolve &) = delete;
    ShiftedSolve &operator=(const ShiftedSolve &) = delete;

    // grid of the per-shift update kernels (sh_vec_shift, lop_vec_update): 256 threads of two rows each
    int update_grid() const { return std::max(1, std::min(c.sm_count * 8, (n + 511) / 512)); }
    template <class T> T *alloc(size_t count)       // device memory of the workspace
    {
        void *p = c.dev_alloc(std::max<size_t>(count * sizeof(T), 16));
        ws.mem.push_back(p);
        return (T *)p;
    }
    // A synchronous solve, before its enqueue half: time the reference's timed region and, with BICG_SHIFT_ERROR, keep b (the
    // caller's r, moved by `in`) for report_error.
    void synchronous(const double *r, cudaMemcpyKind in)
    {
        BICG_CUDA(cudaEventCreate(&e0)); BICG_CUDA(cudaEventCreate(&e1));
        if (in == cudaMemcpyHostToDevice) pcie_bytes = ((uint64_t)L + 1) * n * 8;
        if (c.cfg.shift_error) BICG_CUDA(cudaMemcpyAsync(ws.d_b, r, (size_t)n * sizeof(double), in, st));
    }
    // x_set (L blocks of n) -> ws.d_x and b -> the arena's r, both moved by `in`; sigma -> d_sigma by sigma_in; fresh scalars
    void upload(const double *x_set, const double *r, const double *sigma, double *d_sigma, cudaMemcpyKind in, cudaMemcpyKind sigma_in)
    {
        BICG_CUDA(cudaMemcpy2DAsync(ws.d_x, stride * sizeof(double), x_set, (size_t)n * sizeof(double), (size_t)n * sizeof(double), L,
                                    in, st));
        BICG_CUDA(cudaMemcpyAsync(d_sigma, sigma, L * sizeof(double), sigma_in, st));
        BICG_CUDA(cudaMemcpyAsync(m->vec(V_R), r, (size_t)n * sizeof(double), in, st));
        reset_scalars(m, 0.0, 0, st);
    }
    // The reference's timed region: run.prologue(), then the loop on the device as a WHILE node around the workspace's captured
    // body of U run.iteration() (variant: which of the family's captured loops), at most max_iter / U bodies.
    template <class Run> void run(Run &run, int max_iter, const int *d_done, int v)
    {
        variant = v;
        launches0 = c.launches;
        if (e0) BICG_CUDA(cudaEventRecord(e0, st));
        run.prologue();
        enqueue_while(m, st, (max_iter + U - 1) / U, 0, 0, ws.exec[v],
                      [&](cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps) { return add_loop(g, deps, ndeps, d_done, v); });
        if (e1) BICG_CUDA(cudaEventRecord(e1, st));
    }
    // prepare: U run.iteration() captured into ws.iters[v] (the kernels they launch in ws.kernels[v]), and the executable graph
    // of the WHILE node around them that an uncaptured call launches
    template <class Run> void capture_loop(Run &run, const int *d_done, int v)
    {
        const int launches = c.launches;            // capture is not execution
        BICG_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        for (int u = 0; u < U; ++u) run.iteration();
        BICG_CUDA(cudaStreamEndCapture(st, &ws.iters[v]));
        ws.kernels[v] = c.launches - launches;
        c.launches = launches;
        cudaGraph_t g = nullptr;
        BICG_CUDA(cudaGraphCreate(&g, 0));
        add_loop(g, nullptr, 0, d_done, v);
        BICG_CUDA(cudaGraphInstantiate(&ws.exec[v], g, 0));
        BICG_CUDA(cudaGraphDestroy(g));
    }
    // after run(): x_set and the seed residual r back into the caller's buffers by `out`, in stream order
    void outputs(double *x_set, double *r, cudaMemcpyKind out)
    {
        BICG_CUDA(cudaMemcpy2DAsync(x_set, (size_t)n * sizeof(double), ws.d_x, stride * sizeof(double), (size_t)n * sizeof(double), L,
                                    out, st));
        BICG_CUDA(cudaMemcpyAsync(r, m->vec(V_R), (size_t)n * sizeof(double), out, st));
    }
    // after run() of a synchronous solve: the outputs, then the solver's device state *d_state and the loop's bodies to the host
    template <class State> State finish(double *x_set, double *r, cudaMemcpyKind out, const State *d_state)
    {
        outputs(x_set, r, out);
        State sd{};
        BICG_CUDA(cudaMemcpyAsync(&sd, d_state, sizeof(State), cudaMemcpyDeviceToHost, st));
        Scalars hs;
        BICG_CUDA(cudaMemcpyAsync(&hs, m->d_sc, sizeof(Scalars), cudaMemcpyDeviceToHost, st));
        AsyncLoopState ls;
        BICG_CUDA(cudaMemcpyAsync(&ls, m->d_loop, sizeof(AsyncLoopState), cudaMemcpyDeviceToHost, st));
        BICG_CUDA(cudaStreamSynchronize(st));
        if (hs.error) timeout_fatal(m, "a shifted solve");
        bodies = ls.count;
        BICG_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        return sd;
    }
    // after finish(): the statistics every shifted solver fills alike (the solver adds iters, converged, final_res)
    bicg_stats stats() const
    {
        bicg_stats st{};
        st.loop_ms = ms;
        st.kernel_launches = c.launches - launches0 + bodies * ws.kernels[variant];
        st.h2d_bytes = pcie_bytes; st.d2h_bytes = pcie_bytes;
        return st;
    }
    // The last step of every synchronous shifted solver, after its own printout: with BICG_SHIFT_ERROR, the relative error
    // ||(A + sigma_j I) x_j - b|| / ||b|| of every shift from ws.d_x (collective), kept for bicg_last_shift_error and printed by
    // rank 0 as the reference's DISPLAY_ERROR block does (shifted_switching_solver.c:570-598), `seed` being the seed the solve
    // ended with.  The reference measures against (A + sigma_seed I) 1, the b its drivers build; this is the b passed in.
    // It runs after finish() and after the solver took stats(), so the check's launches and time stay out of kernel_launches and
    // loop_ms, like the reference's check, which runs after its timed region.
    void report_error(const double *sigma, int seed)
    {
        c.last_shift_err.clear();
        if (!c.cfg.shift_error) return;
        c.last_shift_err = shift_relative_errors(m, ws.d_x, stride, ws.d_b, sigma, L);
        if (c.rank != 0 || c.cfg.quiet) return;
        printf("seed(0:seed, 1:shift), sigma, relative error\n");                  // :572
        for (int i = 0; i < L; ++i) {
            if (i == seed) printf("0, %e, %e\n", sigma[i], c.last_shift_err[(size_t)i]);               // :593
            else if (i % 10 == 0) printf("1, %e, %e\n", sigma[i], c.last_shift_err[(size_t)i]);        // :594
        }
        fflush(stdout);
    }

private:
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaGraphNode_t add_loop(cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps, const int *d_done, int v) const
    {
        return add_while_node(m, g, deps, ndeps, d_done, [&](cudaGraph_t body, cudaGraphNode_t *tail) -> size_t {
            BICG_CUDA(cudaGraphAddChildGraphNode(&tail[0], body, nullptr, 0, ws.iters[v]));
            return 1;
        });
    }
};

} // namespace bicg
