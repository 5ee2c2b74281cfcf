// spmv.cu -- fp64 CSR SpMV for sm_90a, one kernel per plan kind, each with two epilogues chosen at compile time:
//  * the solver's (SOLVER): y = A x (+ sigma x) with the dot products of the solver fused into the epilogue and the
//    cross-GPU reduction / scalar recurrence in its tail.  Replaces mult() + MPI_csr_spmv_ovlap() (matrix.c:498-516,
//    428-441) and the my_ddot + MPI_Iallreduce pairs that follow them (solver.c:88-91, 96-102, 238-247, 365-367, 381-385).
//  * the batched multiply's (bicg_matrix_multiply, multiply.cu): y_v = alpha (A + sigma_v I) x_v + beta y_v for NV vectors
//    from one pass over the matrix.  It reads nothing in Scalars, and its tail is only the closing barrier with peers.
//
//  spmv_ws_kernel<LANES, CTHREADS, NV, SOLVER>   (kind 0, the default) -- warp-specialised, TMA-fed
//      Persistent CTAs walk a precomputed tile plan (<= CTHREADS/LANES rows and <= cap entries per tile).
//      One PRODUCER warp streams, per tile, everything the consumers will touch except x itself -- the val[]
//      and col[] slices, the ptr[] slice of the tile's rows and, for the solver, the slices of the epilogue vectors
//      (r#, q, ...) -- from HBM into a multi-stage shared-memory ring with 1-D TMA bulk copies (cp.async.bulk + mbarrier
//      complete_tx; UBLKCP in SASS).  CTHREADS/32 CONSUMER warps wait on the stage's "full" mbarrier, consume
//      it and arrive on its "empty" mbarrier; there is no CTA-wide barrier in the loop, so a slow warp never
//      stalls the others and the only long-latency operation left on a consumer's critical path is the
//      gather x[col] (issued 16 at a time per thread so a row costs one L2 round trip).
//      With LANES = 1 a warp's 32 gathers at step j hit the same stencil offset of 32 consecutive rows -> 2
//      cache lines instead of ~15 for banded matrices, and the row is summed left to right exactly like the
//      reference's scalar loop.  LANES > 1 is for long / irregular rows (shuffle reduction in the group).
//      (Round-1 history: the first version used one __syncthreads per tile and loaded ptr / r# from global
//      inside the loop; ncu showed 76 % of cycles with no eligible warp -- profiles/r01a_first_path.json.)
//
//  spmv_rowsplit_kernel<LANES, NV, SOLVER>       (kind 1)
//      Classic sub-warp-per-row kernel reading val/col straight from global memory; fallback for matrices
//      with rows longer than a stage, and the comparison point for the TMA kernel.
//
// Both sum every row with dev.cuh's row_product, so a row's sum is the same bits in either epilogue and at any NV, and
// both write y exactly once (no zero-fill + accumulate passes as in matrix.c:434-440).
#include "spmv.cuh"

namespace bicg {

namespace {

__device__ __forceinline__ bool needs_tail(const KernelCommon &kc)
{
    return kc.tail.op != TAIL_NONE || kc.tail.signal_halo;
}

// UNR * NV gathers in flight per thread: 16 at LANES = 1, else 8, whatever NV is (at least one entry per pass)
template <int LANES, int NV>
constexpr int row_unr() { return ((LANES == 1 ? 16 : 8) / NV) > 0 ? (LANES == 1 ? 16 : 8) / NV : 1; }

// the solver's epilogue of row `row`: y = rowsum (+ sigma x[row]), then dot[k] += U[row] * V[row] for the fused dots, where
// U and V are epilogue vectors (epi(i): vector i at this row) or the y just computed
template <class Epi>
__device__ __forceinline__ void solver_store(const SpmvArgs &a, int row, double acc, Epi epi, int ndot, double (&dot)[4])
{
    if (a.sigma) acc = fma(*a.sigma, ld_coherent(a.x[0] + row), acc);     // s += sigma p (daxpy after the SpMV)
    a.y[0][row] = acc;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (k < ndot) {
            const double av = a.epi.ia[k] >= 0 ? epi(a.epi.ia[k]) : acc;
            const double bv = a.epi.ib[k] >= 0 ? epi(a.epi.ib[k]) : acc;
            dot[k] = fma(av, bv, dot[k]);
        }
    }
}

// the multiply's epilogue of row `row` for every vector of the launch: t = rowsum (+ sigma_v x_v[row]), y_v = alpha t (+ beta y_v)
template <int NV>
__device__ __forceinline__ void multiply_store(const SpmvArgs &a, int row, const double (&acc)[NV])
{
#pragma unroll
    for (int v = 0; v < NV; ++v) {
        if (v < a.nv) {
            double t = acc[v];
            if (a.sigma) t = fma(a.sigma[v], ld_coherent(a.x[v] + row), t);
            a.y[v][row] = a.beta == 0.0 ? a.alpha * t : fma(a.alpha, t, a.beta * a.y[v][row]);
        }
    }
}

// the solver reduces its dots and runs the scalar recurrence; the multiply's tail is at most the closing barrier with peers
template <bool SOLVER>
__device__ __forceinline__ void spmv_tail(const KernelCommon &kc, double (&dot)[4], double *scratch)
{
    if (!needs_tail(kc)) return;
    if constexpr (SOLVER) {
        block_sum<4>(dot, scratch);
        kernel_tail<4>(kc, dot, scratch);
    } else {
        double none[1] = {0.0};
        kernel_tail<0>(kc, none, scratch);
    }
}

template <int LANES, int CTHREADS, int NV, bool SOLVER>
__global__ void __launch_bounds__(CTHREADS + 32, 1) spmv_ws_kernel(const __grid_constant__ SpmvArgs a)
{
    if constexpr (SOLVER)
        if (a.kc.sc->done) return;

    constexpr int RPT = CTHREADS / LANES;            // rows per tile
    constexpr int NCW = CTHREADS / 32;               // consumer warps
    constexpr int UNR = row_unr<LANES, NV>();

    extern __shared__ __align__(128) unsigned char dyn_smem[];
    __shared__ __align__(8) StageRing<StageHdr> ring;
    __shared__ double scratch[SOLVER ? 32 * 4 : 32];

    const int tid = threadIdx.x;
    const int stages = a.stages;
    const StageLayout L(a.cap, RPT, SOLVER ? SPMV_EPI_SLICES : 0);
    const int my_tiles = (a.ntiles > (int)blockIdx.x) ? (a.ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

    if (tid == 0) ring.init(stages, (unsigned)NCW);
    __syncthreads();

    double dot[4] = {0.0, 0.0, 0.0, 0.0};

    if (tid >= CTHREADS) {
        // ===================================== producer warp ==========================================
        if (tid == CTHREADS) {
            // 8-byte values, 32-bit columns, no L2 policy; the solver streams its epilogue vectors
            const TileFormat<> f{false, false, SOLVER ? a.epi.nvec : 0, {}};
            for (int i = 0; i < my_tiles; ++i) {
                const int t = (int)blockIdx.x + i * (int)gridDim.x;
                const int row0 = a.tile_row[t], row1 = a.tile_row[t + 1];
                const TileWindow w = tile_window(row0, row1, a.tile_nz[t], a.tile_nz[t + 1], f.align());
                const int s = ring.acquire(i, stages);
                ring.hdr[s] = StageHdr{row0, row1, w.a0, w.rowa};
                tile_issue(dyn_smem + (size_t)s * L.bytes(), L, ring.full_bar(s), f, w, TileSrc{a.val, nullptr, nullptr, a.col, a.ptr},
                           [&](int v) { return a.epi.vec[v]; });
            }
        }
    } else {
        // ===================================== consumer warps =========================================
        // The matrix stream is already in flight; make sure the peers' halo values of x have landed before
        // the first gather (the reference's MPI_Wait on the allgather, matrix.c:439).
        if (a.wait_halo) {
            if (tid < 32) {
                const bool ok = halo_wait_epoch(a.kc.comm, a.kc.sc->halo_epoch);
                if (!ok && tid == 0) a.kc.sc->error = 1;
            }
            nbar(1, CTHREADS);
        }
        const int lane = tid % LANES;
        const int row_in_tile = tid / LANES;
        const double *x[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) x[v] = a.x[v];
        const int ndot = SOLVER ? a.epi.ndot : 0;

        for (int i = 0; i < my_tiles; ++i) {
            const int s = ring.wait(i, stages);
            const unsigned char *st = dyn_smem + (size_t)s * L.bytes();
            const double   *sval = L.vals(st);
            const double   *sepi = L.epi(st);
            const unsigned *scol = L.cols(st);
            const unsigned *sptr = L.ptrs(st);
            const StageHdr h = ring.hdr[s];
            const int row = h.row0 + row_in_tile;
            const bool valid = row < h.row1;
            int j = 0, e = 0;
            if (valid) {
                j = (int)(sptr[row - h.rowa] - h.a0) + lane;
                e = (int)(sptr[row - h.rowa + 1] - h.a0);
            }
            double acc[NV];
            row_product<LANES, UNR, NV>([&](int idx) { return sval[idx]; }, [&](int idx) { return scol[idx]; }, x, j, e, acc);
            if (valid && lane == 0) {
                if constexpr (SOLVER) {
                    const int ro = row - h.rowa, prow = L.prow;   // by value: nvcc then forms the slice offsets as it did inline
                    solver_store(a, row, acc[0], [=](int v) { return sepi[v * prow + ro]; }, ndot, dot);
                } else {
                    multiply_store<NV>(a, row, acc);
                }
            }
            ring.release(s);
        }
    }

    spmv_tail<SOLVER>(a.kc, dot, scratch);
}

template <int LANES, int NV, bool SOLVER>
__global__ void __launch_bounds__(256) spmv_rowsplit_kernel(const __grid_constant__ SpmvArgs a)
{
    if constexpr (SOLVER)
        if (a.kc.sc->done) return;
    constexpr int UNR = row_unr<LANES, NV>();
    __shared__ double scratch[SOLVER ? 32 * 4 : 32];
    const int tid = threadIdx.x;
    if (a.wait_halo) {
        if (tid < 32) {
            const bool ok = halo_wait_epoch(a.kc.comm, a.kc.sc->halo_epoch);
            if (!ok && tid == 0) a.kc.sc->error = 1;
        }
        __syncthreads();
    }
    constexpr int RPB = 256 / LANES;
    const int lane = tid % LANES;
    const double *x[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) x[v] = a.x[v];
    const int ndot = SOLVER ? a.epi.ndot : 0;
    double dot[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long base = (long long)blockIdx.x * RPB; base < a.rows; base += (long long)gridDim.x * RPB) {
        const int row = (int)base + tid / LANES;
        const bool valid = row < a.rows;
        unsigned pb = 0, pe = 0;
        if (valid) { pb = a.ptr[row]; pe = a.ptr[row + 1]; }
        double acc[NV];
        if constexpr (SOLVER) {
            // row_product's per-lane order (storage order, one fma each, then lanes_sum) in four-entry passes: on the
            // solver's SpMV with its fused dot this loop is faster than row_product's clamped UNR-entry passes
            const double *__restrict__ val = a.val;
            const unsigned *__restrict__ col = a.col;
            double s = 0.0;
            unsigned j = pb + lane;
            for (; j + 3 * LANES < pe; j += 4 * LANES) {
                const unsigned c0 = col[j], c1 = col[j + LANES], c2 = col[j + 2 * LANES], c3 = col[j + 3 * LANES];
                const double v0 = val[j], v1 = val[j + LANES], v2 = val[j + 2 * LANES], v3 = val[j + 3 * LANES];
                s = fma(v0, ld_coherent(x[0] + c0), s);
                s = fma(v1, ld_coherent(x[0] + c1), s);
                s = fma(v2, ld_coherent(x[0] + c2), s);
                s = fma(v3, ld_coherent(x[0] + c3), s);
            }
            for (; j < pe; j += LANES) s = fma(val[j], ld_coherent(x[0] + col[j]), s);
            acc[0] = lanes_sum<LANES>(s);
        } else {
            // entries relative to the row's first one
            const double *__restrict__ rv = a.val + pb;
            const unsigned *__restrict__ rc = a.col + pb;
            row_product<LANES, UNR, NV>([&](int idx) { return rv[idx]; }, [&](int idx) { return rc[idx]; }, x, lane, (int)(pe - pb), acc);
        }
        if (valid && lane == 0) {
            if constexpr (SOLVER)
                solver_store(a, row, acc[0], [&](int v) { return a.epi.vec[v][row]; }, ndot, dot);
            else
                multiply_store<NV>(a, row, acc);
        }
    }
    spmv_tail<SOLVER>(a.kc, dot, scratch);
}

// the instantiations: NV = 1 with the solver's epilogue, NV in {1, 2, 4, 8} with the multiply's; each over every lanes and,
// for the tile kernel, every consumer-thread count of a plan
template <int NV, bool SOLVER, int LANES>
cudaError_t launch_l(int kind, int threads, int grid, size_t smem, const SpmvArgs &a, cudaStream_t st)
{
    if (kind != 0)         spmv_rowsplit_kernel<LANES, NV, SOLVER><<<grid, 256, 0, st>>>(a);
    else if (threads == 128) spmv_ws_kernel<LANES, 128, NV, SOLVER><<<grid, 128 + 32, smem, st>>>(a);
    else if (threads == 256) spmv_ws_kernel<LANES, 256, NV, SOLVER><<<grid, 256 + 32, smem, st>>>(a);
    else if (threads == 512) spmv_ws_kernel<LANES, 512, NV, SOLVER><<<grid, 512 + 32, smem, st>>>(a);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}
template <int NV, bool SOLVER>
cudaError_t launch_nv(int kind, int lanes, int threads, int grid, size_t smem, const SpmvArgs &a, cudaStream_t st)
{
    switch (lanes) {
    case 1:  return launch_l<NV, SOLVER, 1>(kind, threads, grid, smem, a, st);
    case 2:  return launch_l<NV, SOLVER, 2>(kind, threads, grid, smem, a, st);
    case 4:  return launch_l<NV, SOLVER, 4>(kind, threads, grid, smem, a, st);
    case 8:  return launch_l<NV, SOLVER, 8>(kind, threads, grid, smem, a, st);
    case 16: return launch_l<NV, SOLVER, 16>(kind, threads, grid, smem, a, st);
    case 32: return launch_l<NV, SOLVER, 32>(kind, threads, grid, smem, a, st);
    default: return cudaErrorInvalidValue;
    }
}

template <int NV, bool SOLVER, int LANES>
cudaError_t set_attr_l()
{
    cudaError_t e;
    if ((e = smem_optin(spmv_ws_kernel<LANES, 128, NV, SOLVER>)) != cudaSuccess) return e;
    if ((e = smem_optin(spmv_ws_kernel<LANES, 256, NV, SOLVER>)) != cudaSuccess) return e;
    return smem_optin(spmv_ws_kernel<LANES, 512, NV, SOLVER>);
}
template <int NV, bool SOLVER>
cudaError_t set_attr_nv()
{
    cudaError_t e;
    if ((e = set_attr_l<NV, SOLVER, 1>()) != cudaSuccess) return e;
    if ((e = set_attr_l<NV, SOLVER, 2>()) != cudaSuccess) return e;
    if ((e = set_attr_l<NV, SOLVER, 4>()) != cudaSuccess) return e;
    if ((e = set_attr_l<NV, SOLVER, 8>()) != cudaSuccess) return e;
    if ((e = set_attr_l<NV, SOLVER, 16>()) != cudaSuccess) return e;
    return set_attr_l<NV, SOLVER, 32>();
}

} // namespace

void epi_add_dot(EpiArgs &e, const double *a, const double *b)
{
    auto index_of = [&](const double *p) -> int {
        if (!p) return -1;
        for (int i = 0; i < e.nvec; ++i) if (e.vec[i] == p) return i;
        e.vec[e.nvec] = p;
        return e.nvec++;
    };
    e.ia[e.ndot] = index_of(a);
    e.ib[e.ndot] = index_of(b);
    ++e.ndot;
}

int spmv_setup_attributes()
{
    cudaError_t e;
    if ((e = set_attr_nv<1, true>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_nv<1, false>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_nv<2, false>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_nv<4, false>()) != cudaSuccess) return (int)e;
    return (int)set_attr_nv<8, false>();
}

int launch_spmv(int kind, int lanes, int threads, int grid, size_t smem, bool solver, const SpmvArgs &a, cudaStream_t st)
{
    if (solver) return (int)(a.nv == 1 ? launch_nv<1, true>(kind, lanes, threads, grid, smem, a, st) : cudaErrorInvalidValue);
    // the smallest instantiated NV that holds the launch's vectors
    if (a.nv < 1 || a.nv > MUL_NV_MAX) return (int)cudaErrorInvalidValue;
    if (a.nv == 1) return (int)launch_nv<1, false>(kind, lanes, threads, grid, smem, a, st);
    if (a.nv == 2) return (int)launch_nv<2, false>(kind, lanes, threads, grid, smem, a, st);
    if (a.nv <= 4) return (int)launch_nv<4, false>(kind, lanes, threads, grid, smem, a, st);
    return (int)launch_nv<8, false>(kind, lanes, threads, grid, smem, a, st);
}

} // namespace bicg
