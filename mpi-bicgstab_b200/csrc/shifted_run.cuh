// shifted_run.cuh -- what every shifted solver shares (shifted.cu, shifted_lop.cu).
// Host: the seed system runs on the arena vectors through PhaseLauncher (engine.hpp) with shift_sigma set, so its SpMVs
// compute y = (A + sigma_seed I) x, and tail_store puts the reduced epilogue dots into Scalars::pend[] for the solver's own
// scalar kernels.  ShiftedSolve holds everything around a solver's own device state and kernel sequence: the device memory
// the solve owns, the sigma_len solutions x_j (host x_set: copied into one strided device buffer; device x_set: the caller's
// buffer, updated in place), b in / the seed residual out through the arena's r, the update kernels' grid, the timed loop
// and the statistics every shifted solver reports alike.  An asynchronous solve runs the same enqueue half on the caller's
// stream with the handle's workspace (ShiftWork): x_set, r and sigma staged device to device, the loop as a WHILE node.
// Device: the per-shift scalar recurrence both families evaluate (shift_step) and the row-pair accesses their update
// kernels move x_j and p_j with (ld2, st2, ld2x, st2x).  Each family keeps its own update loop: they apply the six
// coefficients in different orders, and LOP folds the seed's update into its last pass.
#pragma once
#include "engine.hpp"

#include <algorithm>
#include <vector>

namespace bicg {

// the two families behind shifted_solve, which has checked sigma_len and seed: shifted.cu (fixed: shifted_lopbicg, else
// shifted_lopbicg_switching) and shifted_lop.cu (pipe: PIPE-LOP, else LOP); dev: x_set and r are device pointers
int switching_solve(bicg_matrix *m, bool fixed, double *x_set, double *r, const double *sigma, int L, int seed, double tol,
                    int max_iter, bool dev);
int lop_solve(bicg_matrix *m, bool pipe, double *x_set, double *r, const double *sigma, int L, int seed, double tol, int max_iter,
              bool dev);
// The asynchronous side of each family (bicg_shifted_solve_async): *_prepare allocates workspace ws for L shifts and the current
// BICG_SHIFT_MAX_ITER when it is empty and captures the variant's loop when it has not been; *_solve_async enqueues the solve
// on st with ws's buffers (x_set, r, sigma: the caller's device pointers; result, stop_iter: optional device outputs).
void switching_prepare(bicg_matrix *m, ShiftWork &ws, int L);
void switching_solve_async(bicg_matrix *m, ShiftWork &ws, bool fixed, double *x_set, double *r, const double *sigma, int seed,
                           double tol, int max_iter, cudaStream_t st, bicg_shift_result *result, int *stop_iter);
void lop_prepare(bicg_matrix *m, ShiftWork &ws, int L, bool pipe);
void lop_solve_async(bicg_matrix *m, ShiftWork &ws, bool pipe, double *x_set, double *r, const double *sigma, int seed, double tol,
                     int max_iter, cudaStream_t st, bicg_shift_result *result, int *stop_iter);

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

// Rows i, i + 1 (two) or i alone of a vector, as one 16-byte access: the arena vectors and every p_set block start 16-byte
// aligned, and the update kernels give each thread an even i.
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
// The same for a block of x_set, which starts 16-byte aligned (al) or only 8-byte aligned: a caller's device x_set has blocks
// of n doubles from any 8-byte aligned base; then the pair moves as two 8-byte accesses.  i is even, so al depends on the
// block alone and is the same for the whole warp.
__device__ __forceinline__ void ld2x(const double *p, int i, bool two, bool al, double (&v)[2])
{
    if (two && !al) { v[0] = p[i]; v[1] = p[i + 1]; }
    else ld2(p, i, two, v);
}
__device__ __forceinline__ void st2x(double *p, int i, bool two, bool al, const double (&v)[2])
{
    if (two && !al) { p[i] = v[0]; p[i + 1] = v[1]; }
    else st2(p, i, two, v);
}
__device__ __forceinline__ bool aligned16(const double *p) { return (reinterpret_cast<size_t>(p) & 15) == 0; }

struct ShiftedSolve {
    static constexpr int U = 8, DEPTH = 2;   // iterations per batch; batches enqueued ahead of the done flag the host reads
    bicg_matrix *m;
    Context &c;
    const int n, L;
    const bool dev;                          // x_set and r are device pointers: no copy of x_set, r moves device to device
    ShiftWork *const ws;                     // asynchronous solve: the handle's workspace of the family, x_set staged in ws->d_x
    const cudaStream_t st;                   // where the solve is enqueued: the library's stream, or the caller's
    const long long stride;                  // doubles between consecutive shifts in the solver's p_set (16-byte aligned blocks)
    const long long xstride;                 // ... in d_x: stride (host x_set, workspace), n (the caller's device x_set; any alignment)
    double *d_x = nullptr;                   // [L][xstride] the solutions x_j
    double *d_b = nullptr;                   // BICG_SHIFT_ERROR only: the caller's b
    float ms = 0.f;                          // length of the timed region
    int launches0 = 0;
    std::vector<void *> owned;

    // synchronous solve: the library's stream, buffers allocated per call
    ShiftedSolve(bicg_matrix *mm, int sigma_len, bool device_vectors)
        : m(mm), c(ctx()), n(mm->n_loc), L(sigma_len), dev(device_vectors), ws(nullptr), st(ctx().stream),
          stride(((long long)mm->n_loc + 15) / 16 * 16), xstride(device_vectors ? (long long)mm->n_loc : stride) {}
    // asynchronous solve on `s` with the buffers of workspace w (which its prepare allocates through alloc())
    ShiftedSolve(bicg_matrix *mm, int sigma_len, ShiftWork &w, cudaStream_t s)
        : m(mm), c(ctx()), n(mm->n_loc), L(sigma_len), dev(true), ws(&w), st(s), stride(((long long)mm->n_loc + 15) / 16 * 16),
          xstride(stride), d_x(w.d_x) {}
    ~ShiftedSolve() { for (void *p : owned) c.dev_free(p); }
    ShiftedSolve(const ShiftedSolve &) = delete;
    ShiftedSolve &operator=(const ShiftedSolve &) = delete;

    // grid of the per-shift update kernels (sh_vec_shift, lop_vec_update): 256 threads of two rows each
    int update_grid() const { return std::max(1, std::min(c.sm_count * 8, (n + 511) / 512)); }
    template <class T> T *alloc(size_t count)       // device memory freed when the solve ends, or the workspace's
    {
        void *p = c.dev_alloc(std::max<size_t>(count * sizeof(T), 16));
        (ws ? ws->mem : owned).push_back(p);
        return (T *)p;
    }
    // x_set (L blocks of n) -> d_x (device x_set: d_x is x_set; asynchronous: the workspace's), sigma -> d_sigma, b -> the arena's
    // r, fresh solver scalars
    void upload(double *x_set, const double *r, const double *sigma, double *d_sigma)
    {
        if (ws) {
            BICG_CUDA(cudaMemcpy2DAsync(d_x, stride * sizeof(double), x_set, (size_t)n * sizeof(double), (size_t)n * sizeof(double),
                                        L, cudaMemcpyDeviceToDevice, st));
        } else if (dev) {
            d_x = x_set;
        } else {
            d_x = alloc<double>((size_t)L * stride);
            BICG_CUDA(cudaMemcpy2DAsync(d_x, stride * sizeof(double), x_set, (size_t)n * sizeof(double), (size_t)n * sizeof(double),
                                        L, cudaMemcpyHostToDevice, st));
        }
        BICG_CUDA(cudaMemcpyAsync(d_sigma, sigma, L * sizeof(double), ws ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        BICG_CUDA(cudaMemcpyAsync(m->vec(V_R), r, (size_t)n * sizeof(double), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                                  st));
        if (!ws && c.cfg.shift_error) {
            d_b = alloc<double>(n);
            BICG_CUDA(cudaMemcpyAsync(d_b, m->vec(V_R), (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
        }
        reset_scalars(m, 0.0, 0, st);
    }
    // The reference's timed region: run.prologue(), then batches of U run.iteration() until the device raises *d_done.
    // Synchronous: the host enqueues the batches and polls the flag (run_batches).  Asynchronous: the loop runs on the device
    // as a WHILE node around the workspace's captured batch (variant: which of the family's captured loops), with the same bound.
    template <class Run> void run(Run &run, int max_iter, const int *d_done, int variant)
    {
        if (ws) {
            run.prologue();
            enqueue_while(m, st, (max_iter + U - 1) / U, 0, 0, ws->exec[variant],
                          [&](cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps) { return add_loop(g, deps, ndeps, d_done, variant); });
            return;
        }
        BICG_CUDA(cudaEventCreate(&e0)); BICG_CUDA(cudaEventCreate(&e1));
        launches0 = c.launches;
        BICG_CUDA(cudaEventRecord(e0, st));
        run.prologue();
        run_batches(max_iter, U, DEPTH, d_done, [&](int) { for (int u = 0; u < U; ++u) run.iteration(); });
        BICG_CUDA(cudaEventRecord(e1, st));
    }
    // prepare of an asynchronous solve: U run.iteration() captured into ws->iters[variant], and the executable graph of the
    // WHILE node around them that an uncaptured call launches
    template <class Run> void capture_loop(Run &run, const int *d_done, int variant)
    {
        const int launches = c.launches;            // capture is not execution
        BICG_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        for (int u = 0; u < U; ++u) run.iteration();
        BICG_CUDA(cudaStreamEndCapture(st, &ws->iters[variant]));
        c.launches = launches;
        cudaGraph_t g = nullptr;
        BICG_CUDA(cudaGraphCreate(&g, 0));
        add_loop(g, nullptr, 0, d_done, variant);
        BICG_CUDA(cudaGraphInstantiate(&ws->exec[variant], g, 0));
        BICG_CUDA(cudaGraphDestroy(g));
    }
    // after run(): x_set (host x_set only), the seed residual r and the solver's device state *d_state back to the host
    template <class State> State finish(double *x_set, double *r, const State *d_state)
    {
        if (!dev)
            BICG_CUDA(cudaMemcpy2DAsync(x_set, (size_t)n * sizeof(double), d_x, stride * sizeof(double), (size_t)n * sizeof(double), L,
                                        cudaMemcpyDeviceToHost, st));
        BICG_CUDA(cudaMemcpyAsync(r, m->vec(V_R), (size_t)n * sizeof(double), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                                  st));
        State out{};
        BICG_CUDA(cudaMemcpyAsync(&out, d_state, sizeof(State), cudaMemcpyDeviceToHost, st));
        Scalars hs;
        BICG_CUDA(cudaMemcpyAsync(&hs, m->d_sc, sizeof(Scalars), cudaMemcpyDeviceToHost, st));
        BICG_CUDA(cudaStreamSynchronize(st));
        if (hs.error) fatal("bicgstab_b200: rank %d timed out waiting for a peer GPU in the shifted solver", m->rank);
        BICG_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        return out;
    }
    // after run() of an asynchronous solve: x_set and r back into the caller's buffers, in stream order
    void finish_async(double *x_set, double *r)
    {
        BICG_CUDA(cudaMemcpy2DAsync(x_set, (size_t)n * sizeof(double), d_x, stride * sizeof(double), (size_t)n * sizeof(double), L,
                                    cudaMemcpyDeviceToDevice, st));
        BICG_CUDA(cudaMemcpyAsync(r, m->vec(V_R), (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
    // after finish(): the statistics every shifted solver fills alike (the solver adds iters, converged, final_res)
    bicg_stats stats() const
    {
        bicg_stats st{};
        st.loop_ms = ms;
        st.kernel_launches = c.launches - launches0;
        st.h2d_bytes = dev ? 0 : (uint64_t)L * n * 8 + (uint64_t)n * 8; st.d2h_bytes = st.h2d_bytes;
        return st;
    }
    // The last step of every shifted solver, after its own printout: with BICG_SHIFT_ERROR, the relative error
    // ||(A + sigma_j I) x_j - b|| / ||b|| of every shift from d_x (collective), kept for bicg_last_shift_error and printed by
    // rank 0 as the reference's DISPLAY_ERROR block does (shifted_switching_solver.c:570-598), `seed` being the seed the solve
    // ended with.  The reference measures against (A + sigma_seed I) 1, the b its drivers build; this is the b passed in.
    // It runs after finish() and after the solver took stats(): d_x lives until the ShiftedSolve is destroyed (or is the
    // caller's x_set), a host x_set is already a copy of it, and the check's launches and time stay out of kernel_launches and loop_ms, like the reference's
    // check, which runs after its timed region.
    void report_error(const double *sigma, int seed)
    {
        c.last_shift_err.clear();
        if (!d_b) return;
        c.last_shift_err = shift_relative_errors(m, d_x, xstride, d_b, sigma, L);
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
    cudaGraphNode_t add_loop(cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps, const int *d_done, int variant) const
    {
        return add_while_node(m, g, deps, ndeps, d_done, [&](cudaGraph_t body, cudaGraphNode_t *tail) -> size_t {
            BICG_CUDA(cudaGraphAddChildGraphNode(&tail[0], body, nullptr, 0, ws->iters[variant]));
            return 1;
        });
    }
};

} // namespace bicg
