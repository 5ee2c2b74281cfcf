// engine.hpp -- host-side runtime of libbicgstab_b200: process context, device-resident matrix, solver driver.
#pragma once
#include "bicgstab_b200.h"
#include "dev.cuh"
#include "plan.hpp"
#include "spmv.cuh"
#include "vec.cuh"
#include "mega.cuh"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <initializer_list>
#include <map>
#include <string>
#include <vector>

namespace bicg {

[[noreturn]] void fatal(const char *fmt, ...);
#define BICG_CUDA(call)                                                                              \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            ::bicg::fatal("bicgstab_b200: CUDA error %s at %s:%d: %s", cudaGetErrorName(e_), __FILE__, \
                          __LINE__, cudaGetErrorString(e_));                                          \
    } while (0)

struct Config {
    double tol = 1.0e-15;        // solver.c:3
    int max_iter = 1000;         // solver.c:4
    int out_iter = 100;          // solver.c:9
    int quiet = 0;
    int spmv_kind = -1;          // -1 auto, 0 tma, 1 rowsplit
    int spmv_lanes = 0;          // 0 choose
    int spmv_threads = 0;
    int spmv_stages = 0;
    int spmv_ctas = 0;           // CTAs per SM (0 choose)
    int autotune = 1;
    int unroll = 10;
    int cache = 1;
    int mega = 1;                // 1: persistent cooperative kernel for the iteration loop where applicable
    int mega_threads = 0;        // 0 choose (512, else 256)
    int mega_trace = 0;
    int mega_lanes = 0;          // lanes per row of the persistent kernel's SpMV (0 choose from the mean row length)
    int resident = 1;            // persistent kernel: keep a CTA's matrix slice in shared memory for the whole solve when it fits
    int row_weight = 1200;       // per-row cost (byte equivalents) next to 24 B per entry when CTA row ranges are balanced
    int boundary_weight = 300;   // extra work (bytes) charged per pushed row when CTA row ranges are balanced
    int device = -1;
    int halo_gap = 64;
    int verbose = 0;
    double shift_tol = 1.0e-12;  // EPS of the shifted solvers (shifted_switching_solver.c:5)
    int shift_max_iter = 1000;   // their MAX_ITER (:6)
    int shift_error = 0;         // 1: after a shifted solve, the relative error of every shift (their DISPLAY_ERROR, :17)
    int peer_timeout_s = 20;     // bound of device-side waits for peers / other CTAs (then: error + exit(1))
};

struct TuneKey {
    int n_loc; size_t nnz; unsigned max_row; int kind;
    bool operator<(const TuneKey &o) const
    {
        if (n_loc != o.n_loc) return n_loc < o.n_loc;
        if (nnz != o.nnz) return nnz < o.nnz;
        if (max_row != o.max_row) return max_row < o.max_row;
        return kind < o.kind;
    }
};
struct TuneVal { int kind, lanes, threads, stages, ctas; };

struct Context {
    bool ready = false;
    Config cfg;
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    // job
    int rank = 0, world = 1;
    bicg_allgather_fn allgather = nullptr;
    void *allgather_ctx = nullptr;
    // results of the last solve
    std::vector<double> last_hist;
    bicg_stats last_stats{};
    std::vector<int> last_shift_stop;     // shifted solver: iteration at which every shift stopped
    int last_shift_seed = 0;              // ... and the seed it ended with
    std::vector<double> last_shift_err;   // BICG_SHIFT_ERROR: ||(A + sigma_j I) x_j - b|| / ||b|| of the last shifted solve
    // host-pointer keyed cache of uploaded matrices
    std::map<const void *, bicg_matrix *> cache;
    std::map<TuneKey, TuneVal> tuned;     // SpMV autotune winners by matrix shape
    // profiling of individual launches
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int> prof_class;
    int launches = 0;

    void ensure();               // lazy device init; fails loudly if there is no usable GPU
    // device-memory cache: cudaMalloc / cudaFree are synchronising driver calls that cost milliseconds for the
    // 100 MB-class buffers of a matrix; blocks are kept by exact size and reused by the next upload
    void *dev_alloc(size_t bytes);
    void  dev_free(void *p);
    void  dev_release_all();
    void  dev_free_after(std::initializer_list<void *> ptrs, cudaEvent_t ev);   // dev_free once `ev` has completed
    void  dev_sweep(bool wait);
    struct Deferred { cudaEvent_t ev; std::vector<void *> ptrs; };
    std::vector<Deferred> deferred;
    std::multimap<size_t, void *> pool;
    std::map<void *, size_t> live;
    size_t pool_bytes = 0;
    // IPC-exported arenas (world > 1) are never freed between matrices: an un-cached call (BICG_CACHE=0) re-uses a parked
    // arena of the same size, and the peers keep their mappings, so no cudaMalloc / cudaIpcOpenMemHandle /
    // cudaIpcCloseMemHandle sits in the reference-facing call after the first one
    struct ArenaRec { char *ptr; size_t bytes; unsigned long long id; cudaIpcMemHandle_t handle; };
    std::multimap<size_t, ArenaRec> arena_pool;
    std::map<std::pair<int, unsigned long long>, void *> peer_maps;    // (rank, that rank's arena id) -> mapped base
    unsigned long long next_arena_id = 1;
    void release_arenas();       // collective: unmap the peers' arenas, free the parked ones
    void host_allgather(const void *send, void *recv, size_t bytes);
    // Host -> device copy ordered on `stream`.  Pinned sources go straight to cudaMemcpyAsync.  Large PAGEABLE sources (what the
    // reference's main.c passes: plain malloc, main.c:81-107) are staged by a few host threads through pinned bounce buffers, each
    // thread copying and issuing its own chunks -- the driver's own pageable path stages with one thread (~11 GB/s).
    void h2d(void *dst, const void *src, size_t bytes);
    struct Stager { cudaStream_t st = nullptr; cudaEvent_t ev[2] = {nullptr, nullptr}; cudaEvent_t done = nullptr; char *buf[2] = {nullptr, nullptr}; };
    std::vector<Stager> stagers;
    int stage_threads = 4;
};
Context &ctx();
void load_config_from_env(Config &c);                              // every option of matrix.cu's table set as BICG_<key>
int  set_option(Config &c, const char *key, const char *value);    // -1: unknown key


struct SpmvPlan {
    int kind = 0, lanes = 1, threads = 256, stages = 3, cap = 0, grid = 0, ctas_per_sm = 1;
    size_t smem = 0;
    int ntiles = 0;
    int *d_tile_row = nullptr;
    unsigned *d_tile_nz = nullptr;
    double ms = 0.0;             // measured time of one launch (autotune) or 0
};

struct MegaPlan {
    bool ok = false;
    int threads = 512, lanes = 1, stages = 2, cap = 0, grid = 0;
    size_t smem = 0;
    size_t res_smem = 0;         // > 0: every CTA's slice fits into shared memory (mega_resident_bytes of the largest one)
    int ntiles = 0;
    int *d_tile_row = nullptr;
    unsigned *d_tile_nz = nullptr;
    int *d_cta_tile = nullptr;
    int4 *d_cta_dep = nullptr;
    unsigned short *d_col16 = nullptr;   // nnz + 16: 16-bit column codes of the CTAs whose column window fits them (mega.cu)
    bool stream_codes = true;    // streaming CTAs use d_col16 where they can (false: 32-bit columns; bicg_debug_stream_codes)
    ValTable *d_vtab = nullptr;  // grid: every CTA's value table (mega.cu: mega_value_kernel)
    unsigned char *d_vhi = nullptr;      // nnz + 16 each: the packed values of the CTAs that have codes and a value table
    unsigned short *d_vmid = nullptr;
    unsigned *d_vlo = nullptr;
    bool stream_values = true;   // those CTAs stream the packed values (false: 8-byte values; bicg_debug_stream_values)
    int *d_tile_flag = nullptr;  // only when rows longer than a stage were cut into chunk tiles
    bool chunked = false;
    std::vector<int> cta_row;    // grid + 1: first row of every CTA
};

// The kernel-per-phase loop of a solve (solve.cu): the captured bodies, the kernels each launches, and the executable graph of
// one WHILE node around them that an uncaptured call launches.
// device memory: bodies run (PIPE_RR: iterations run), their bound, PIPE_RR's schedule, what the last body added to count
struct AsyncLoopState { int count, batches, krr, nrr, step; };
struct AsyncLoop {
    cudaGraph_t iters = nullptr;      // `unroll` iterations (PIPE_RR: `unroll` pipe_iter)
    cudaGraph_t one = nullptr;        // PIPE_RR: one pipe_iter
    cudaGraph_t rr = nullptr;         // PIPE_RR: one rr_replace_iter
    cudaGraphExec_t exec = nullptr;
    int unroll = 0;
    int kernels = 0, kernels_one = 0, kernels_rr = 0;  // kernels of one run of iters / one / rr
};

// What a shifted solve of one family (shifted.cu, shifted_lop.cu) keeps on a handle: every device buffer of the solve for
// sigma_len = L and BICG_SHIFT_MAX_ITER up to cap, its state template, and per variant of the family the captured body of
// ShiftedSolve::U iterations, the kernels it launches and the executable graph of one WHILE node around it.
struct ShiftWork {
    int L = 0, cap = 0;
    std::vector<void *> mem;             // every buffer below and the family's arrays (Context::dev_alloc)
    void *d_state = nullptr;             // ShiftDev / LopDev
    void *d_tmpl = nullptr;              // the same with its pointers and L set, copied into d_state at every solve's start
    std::vector<unsigned char> tmpl;     // host copy of *d_tmpl (the buffers the enqueue stages sigma into and clears)
    double *d_x = nullptr;               // [L][stride] the caller's x_set, staged
    double *d_p = nullptr;               // [L][stride] p_j
    double *d_b = nullptr;               // [n] b, kept by a synchronous solve for BICG_SHIFT_ERROR
    cudaGraph_t iters[2] = {};
    cudaGraphExec_t exec[2] = {};
    int kernels[2] = {};
};
// where the last asynchronous shifted solve on a handle left its history (device memory, written by its result kernel)
struct ShiftHistRef { const double *hist; int n, pad; };
// one value a transpose refresh pushes to a peer: the source's d_val[src] into slot `slot` of rank `rank`'s receive region
struct TransposePush { int src, rank, slot; };

} // namespace bicg

// the opaque handle of the C ABI
struct bicg_matrix {
    int rank = 0, world = 1;
    int n_loc = 0, n_glob = 0;
    size_t nnz = 0;              // entries of this rank's rows (diag + offd)
    size_t nnz_offd = 0;         // ... of them from the offd block (0 on one rank)
    unsigned max_row = 0;
    double mean_row = 0.0;
    // device CSR over the extended local column space
    double *d_val = nullptr;
    unsigned *d_col = nullptr;
    unsigned *d_ptr = nullptr;
    // value updates (bicg_matrix_set_values*, bicg_matrix_shift_diagonal): with offd entries, the diag and offd row pointers of
    // the creation, [2][n_loc + 1], which place the caller's values in d_val; the position in d_val of every own row's
    // diagonal entry (-1: none), computed at the first shift, and whether some row has none
    unsigned *d_blk_ptr = nullptr;
    int *d_diag_pos = nullptr;
    bool diag_missing = false;
    // bicg_matrix_shift_diagonal_async_prepare has run, and whether it found a row without a diagonal entry on some rank
    bool diag_prepared = false, diag_refused = false;
    // test hooks of the value gradient (bicg_debug_value_grad_layout): a forced group width per row (0: chosen) and, at one
    // rank, caller-supplied diag / offd row pointers [2][n_loc + 1] that split every merged row (null: the handle's own order)
    int vg_lanes = 0;
    const unsigned *vg_blk_ptr = nullptr;
    bicg::SpmvPlan plan;
    bicg::MegaPlan mega;             // persistent-kernel plan (mega.cu)
    bicg::MegaSync *d_msync = nullptr;
    bicg::MegaSync *peer_msync[bicg::MAX_RANKS] = {};
    unsigned long long *d_ll = nullptr;                      // LL halo regions [3][ll_stride][2 words] (world > 1)
    long long ll_stride = 0;
    unsigned long long *peer_ll[bicg::MAX_RANKS] = {};
    long long peer_ll_stride[bicg::MAX_RANKS] = {};
    unsigned long long *d_trace = nullptr;   // BICG_MEGA_TRACE
    // ghost layout
    int ghost_off = 0;           // first ghost column index = roundup(n_loc, 16)
    int n_ghost = 0;
    long long vstride = 0;       // doubles between consecutive arena vectors
    std::vector<int> recv_runs;  // quadruples (first_col, len, owner, ghost_idx)
    // arena (one cudaMalloc, IPC-shared with the peers)
    char *arena = nullptr;
    size_t arena_bytes = 0;
    unsigned long long arena_id = 0;         // world > 1: identity of the exported allocation
    cudaIpcMemHandle_t arena_handle{};
    double *vec_base = nullptr;
    bicg::Scalars *d_sc = nullptr;
    double *d_partials = nullptr;
    double *d_hist = nullptr;
    double *hist_extra = nullptr;   // replaces the arena slot when BICG_MAX_ITER grows
    int hist_cap = 0;
    bicg::Mailbox *d_mail = nullptr;
    bicg::HaloFlag *d_hflag = nullptr;
    bicg::CommDev comm{};
    // peers
    void *peer_base[bicg::MAX_RANKS] = {};
    long long peer_vec_off[bicg::MAX_RANKS] = {}, peer_vstride[bicg::MAX_RANKS] = {}, peer_ghost_off[bicg::MAX_RANKS] = {};
    int npush = 0;                                   // peers this rank sends to
    int push_peer[bicg::MAX_RANKS - 1] = {};
    bicg::PushRun *d_push_runs[bicg::MAX_RANKS - 1] = {};
    int push_nruns[bicg::MAX_RANKS - 1] = {};
    // fused-vector launch shape
    int vgrid = 0, vchunk = 0;
    // cache key
    const void *host_key = nullptr;
    uint64_t host_fp = 0;            // content fingerprint of the caller's arrays at upload time (matrix.cu)
    double upload_ms = 0.0;
    cudaEvent_t ev_upload0 = nullptr, ev_upload1 = nullptr;   // around upload + planning; read lazily (matrix_upload_ms)
    uint64_t upload_bytes = 0;
    // asynchronous solves (bicg_solve_async): the last work they enqueued on this handle, which every later call waits for,
    // the device state of their loop, and per method what bicg_solve_async_prepare built
    cudaEvent_t ev_last = nullptr;
    bicg::AsyncLoopState *d_loop = nullptr;
    bicg::AsyncLoop async[4];
    bool captured = false;                // a caller has captured a solve on this handle into a graph
    std::vector<double *> hist_retired;   // histories replaced while such a graph may still write them
    // asynchronous shifted solves (bicg_shifted_solve_async): one workspace per family (0: switching / fixed seed, 1: LOP),
    // buffers of workspaces replaced while a captured graph may still use them, and the history of the last such solve
    bicg::ShiftWork shift_ws[2];
    std::vector<void *> shift_retired;
    bicg::ShiftHistRef *d_shift_last = nullptr;
    // identity of the handle (never reused in a process): what a transpose records as its source
    unsigned long long uid = 0;
    // a handle made by bicg_matrix_create_transpose (transpose.cu): the source's uid; for every entry of d_val the position
    // in the source's d_val it is copied from (>= 0) or ~slot of the receive region (< 0); the source's entries that other
    // ranks hold in their transposes, pushed by a refresh into those ranks' receive regions; and this rank's receive region
    // in the arena (t_nrecv doubles) with every peer's, as mapped here
    unsigned long long t_src_uid = 0;
    int *d_tperm = nullptr;
    bicg::TransposePush *d_tpush = nullptr;
    int t_npush = 0;
    double *d_trecv = nullptr;
    size_t t_nrecv = 0;
    double *peer_trecv[bicg::MAX_RANKS] = {};
    // the same tables over the block orders set_values takes, for bicg_matrix_transpose_entries_async (an entry's block index
    // is j for diag entry j, diag nz + j for offd entry j; they alias d_tperm / d_tpush where block and merged order agree):
    // d_tbperm[b] is the source block index entry b of this handle is copied from (>= 0) or ~slot; d_tbpush pushes source
    // block indices.  The reverse direction: d_trpush sends each received entry (src: this handle's block index) back to the
    // reverse region of the source's rank, at d_trecv + t_rev_off there, whose entry e belongs to source block index
    // d_trev_src[e] (e < t_npush: the entries this rank pushes forward, in push order)
    int *d_tbperm = nullptr;
    bicg::TransposePush *d_tbpush = nullptr;
    bicg::TransposePush *d_trpush = nullptr;
    int t_nrpush = 0;
    int *d_trev_src = nullptr;
    size_t t_rev_off = 0;
    // bicg_matrix_multiply_values_async: caller weights staged into merged order (nnz + 16 doubles), where they cannot be read
    // in place; allocated by bicg_matrix_multiply_values_async_prepare
    double *d_wval = nullptr;

    double *vec(int id) const { return vec_base + (long long)id * vstride; }
};

namespace bicg {

// matrix.cu.  recv_doubles > 0: the arena also holds a region of that many doubles that the peers can store into (the receive
// region of a transpose, transpose.cu), at m->d_trecv, and m->peer_trecv[p] is rank p's
bicg_matrix *matrix_create(const CSR_Matrix *diag, const CSR_Matrix *offd, const INFO_Matrix *info, size_t recv_doubles = 0);
void matrix_destroy(bicg_matrix *m);
double matrix_upload_ms(bicg_matrix *m);
bicg_matrix *matrix_get_cached(const CSR_Matrix *diag, const CSR_Matrix *offd, const INFO_Matrix *info, bool *fresh);
// the persistent kernel's value tables and packed values from d_val, on st: what creation and every value update run last
void launch_value_tables(const bicg_matrix *m, cudaStream_t st);
// device values in the block order set_values takes -> out in m's merged order (nnz doubles), on st
void merge_values(const bicg_matrix *m, const double *diag_val, const double *offd_val, double *out, cudaStream_t st);
// [a, a + abytes) and [b, b + bbytes) overlap; an empty range counts as one byte
inline bool overlaps(const void *a, size_t abytes, const void *b, size_t bbytes)
{
    const uintptr_t a0 = (uintptr_t)a, b0 = (uintptr_t)b;
    return a0 < b0 + std::max<size_t>(bbytes, 1) && b0 < a0 + std::max<size_t>(abytes, 1);
}
// solve.cu
int  solve(bicg_matrix *m, int method, double *x, double *r, int krr, int nrr, int device_vectors, bicg_stats *st);

// calls.cu: what the entry points on a handle do around their work.
// Every synchronous entry point that touches a handle first makes the library's stream wait for the handle's last
// asynchronous work (free when there is none).
void wait_handle(bicg_matrix *m);
// the handle's first asynchronous use: creates its last-work event, recorded on the library's stream
void async_handle_init(bicg_matrix *m);
bool capturing(cudaStream_t st);           // st is capturing into a graph
// An asynchronous call's work on st: st waits for the last work of every handle, enqueue() runs, and its work becomes the
// last work of every handle.  captured: the wait and the record are external nodes of the capture, so that every replay waits
// for the handles' last work at replay time and later calls wait for the replay.
void stream_ordered(std::initializer_list<bicg_matrix *> handles, cudaStream_t st, bool captured, const std::function<void()> &enqueue);
// Collective, host only: false on every rank when any rank is bad or passed other `same` values than this one.  A rank with bad
// arguments must not leave the others waiting for it in collective work on the device.
bool ranks_agree(bool bad, std::initializer_list<long long> same);
// a device-side wait for a peer or another CTA timed out (Scalars::error) during the operation `during`: exit(1)
[[noreturn]] void timeout_fatal(const bicg_matrix *m, const char *during);
// the end of a synchronous call: synchronises the library's stream, then timeout_fatal if m's Scalars::error is set
void sync_checked(bicg_matrix *m, const char *during);

void drop_async_loop(AsyncLoop &L);        // frees the prepared kernel-per-phase loop of one method
// The device-side loop of every kernel-per-phase solve, shared by solve.cu and the shifted solvers.
cudaGraphNode_t add_kernel_node(cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps, const void *fn, void **args);
cudaGraphNode_t add_conditional_node(cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps, cudaGraphConditionalHandle h,
                                     cudaGraphConditionalNodeType type, cudaGraph_t *body);
// A WHILE node of g behind deps: `fill` adds the body's work to `body` and returns its last nodes (at most 3) in `tail`; then
// loop_next_kernel runs the body again unless *done is set or m->d_loop's bound of bodies has run (allocates m->d_loop)
cudaGraphNode_t add_while_node(bicg_matrix *m, cudaGraph_t g, const cudaGraphNode_t *deps, size_t ndeps, const int *done,
                               const std::function<size_t(cudaGraph_t body, cudaGraphNode_t *tail)> &fill);
// the loop on `st` without the host: loop_begin_kernel (`batches` bodies at most), then the node `add` builds into the caller's
// capture, or else the prepared executable graph `exec` of that node
void enqueue_while(bicg_matrix *m, cudaStream_t st, int batches, int krr, int nrr, cudaGraphExec_t exec,
                   const std::function<cudaGraphNode_t(cudaGraph_t, const cudaGraphNode_t *, size_t)> &add);
void drop_shift_work(bicg_matrix *m);      // matrix_destroy: every workspace, its graphs and the retired buffers (shifted.cu)
int  spmv_host(bicg_matrix *m, const double *x_loc, double *y_loc, double *x_full_or_null);
void print_reference_lines(const bicg_stats &st, const std::vector<double> &hist);
void print_times(double seconds, double iters);          // "Total time" / "Avg time/iter" (= seconds / iters), then flush
void reset_scalars(bicg_matrix *m, double tol, int max_iter);   // Scalars of a new solve (enqueued on the stream)
void reset_scalars(bicg_matrix *m, double tol, int max_iter, cudaStream_t st);
// shifted.cu: method = BICG_SHIFTED_*, with BICG_SHIFT_TOL and BICG_SHIFT_MAX_ITER; returns what that solver returns
// (shifted_lopbicg_switching: iterations + 1, the others: the iterations performed), -1 for an unknown method, sigma_len <= 0
// or seed outside [0, sigma_len).  device_vectors: x_set (sigma_len blocks of n_loc, any 8-byte alignment) and r are device
// pointers, else host pointers; sigma is always a host array.
int  shifted_solve(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, int seed,
                   bool device_vectors);
// shift_check.cu, collective: x_j = d_x + j ldx (own rows, device), d_b (device), sigma (host) -> sum_i ((A + sigma_j I) x_j - b)_i^2
// for j < L and sum_i b_i^2 last (L + 1 values, over every rank, added in rank order); enqueued on the stream, synchronises
std::vector<double> shift_residual_sums(bicg_matrix *m, const double *d_x, long long ldx, const double *d_b, const double *sigma, int L);
// ... as ||(A + sigma_j I) x_j - b|| / ||b||
std::vector<double> shift_relative_errors(bicg_matrix *m, const double *d_x, long long ldx, const double *d_b, const double *sigma, int L);
// an empty cross-GPU reduction on st: every rank has finished what it enqueued on the handle before (with peers only)
void peer_barrier(bicg_matrix *m, cudaStream_t st);
// helpers shared by matrix.cu / solve.cu
SpmvArgs make_spmv_args(const bicg_matrix *m, const SpmvPlan &p, int x_id, int y_id);
void launch_spmv_plan(const bicg_matrix *m, const SpmvPlan &p, const SpmvArgs &a, cudaStream_t st, int prof_class = 0);

// reduction tails of the kernel-per-phase kernels
inline TailDesc tail_none() { return TailDesc{TAIL_NONE, FIN_NONE, 0, 0, 0, 0, 0}; }
inline TailDesc tail_allreduce(int fin, int ndot, int npend = 0) { return TailDesc{TAIL_ALLREDUCE, fin, ndot, npend, 0, 0, 0}; }
inline TailDesc tail_post(int ndot) { return TailDesc{TAIL_POST, FIN_NONE, ndot, 0, 0, 0, 0}; }
inline TailDesc tail_complete(int fin, int nred) { return TailDesc{TAIL_COMPLETE, fin, 0, 0, 0, nred, 0}; }
inline TailDesc tail_pend(int ndot, int off) { return TailDesc{TAIL_PEND, FIN_NONE, ndot, 0, off, 0, 0}; }
inline TailDesc tail_store(int ndot) { return TailDesc{TAIL_ALLREDUCE, FIN_STORE_PEND, ndot, 0, 0, 0, 0}; }   // -> Scalars::pend[]

// Kernel-per-phase launcher (solve.cu): one fused vector kernel or one SpMV on the arena vectors per call, each with its
// reduction tail.  The un-shifted loops of solve.cu and the shifted solvers (shifted.cu, shifted_lop.cu) share it.
struct PhaseLauncher {
    bicg_matrix *m;
    Context &c;
    const double *shift_sigma = nullptr;   // device scalar sigma: every SpMV computes y = (A + sigma I) x; null: y = A x
    int launches = 0;                      // kernels launched through vec / spmv (a graph capture takes them back out)
    cudaStream_t stream;                   // where they go: the library's stream unless an asynchronous solve names another

    explicit PhaseLauncher(bicg_matrix *mm) : m(mm), c(ctx()), stream(c.stream) {}
    PhaseLauncher(bicg_matrix *mm, cudaStream_t st) : m(mm), c(ctx()), stream(st) {}
    VecPtrs ptrs() const;
    KernelCommon common(TailDesc tail) const;
    // the boundary runs of arena vector `id` into its ghost slots on the peers; push_src: take the values from there instead
    PushDesc make_push(int id, const double *push_src = nullptr) const;
    // one fused vector kernel; push_vec >= 0: that vector is the next SpMV's input (PH_PUSH: the push alone)
    void vec(int phase, TailDesc tail, int push_vec = -1, const double *push_src = nullptr);
    // y = A x (+ sigma x) with ndot (0..4) epilogue dots (a_k, b_k); a null b_k is the y just computed
    void spmv(int x_id, int y_id, TailDesc tail, int ndot = 0, const double *a0 = nullptr, const double *b0 = nullptr,
              const double *a1 = nullptr, const double *b1 = nullptr, const double *a2 = nullptr, const double *b2 = nullptr,
              const double *a3 = nullptr, const double *b3 = nullptr);
};

// The halo staging of the batched kernels that gather vectors over the extended column space, up to MUL_NV_MAX per launch:
// the multiply (multiply.cu) and the value gradient (value_grad.cu).  The constructor enqueues on st what precedes the first
// batch: with peers, an empty cross-GPU reduction, after which no peer still reads the slots' ghost tails.  stage(x, j0, nv,
// xs) sets xs[v] to x_{j0+v} (x: blocks of n_loc doubles; slots v >= nv repeat the last): the caller's vector at one rank;
// with peers the arena vector MUL_SLOT[v], into which x_{j0+v}'s own rows are copied and whose boundary runs are pushed to the
// neighbours.  Each batch's kernel then waits for the halo flags when wait_halo is set and ends with the tail of kc: with
// peers an empty cross-GPU reduction, so no rank pushes the next batch into a slot a peer is still reading.
struct HaloBatches {
    bicg_matrix *m;
    PhaseLauncher pl;
    bool peers;
    KernelCommon kc;
    int wait_halo;
    HaloBatches(bicg_matrix *m, cudaStream_t st);
    void stage(const double *x, int j0, int nv, const double *(&xs)[MUL_NV_MAX]);
};

} // namespace bicg
