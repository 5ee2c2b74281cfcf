// spmv.cu -- fp64 CSR SpMV for sm_90a with the dot products of the solver fused into its epilogue and the
// cross-GPU reduction / scalar recurrence in its tail.  Replaces mult() + MPI_csr_spmv_ovlap()
// (matrix.c:498-516, 428-441) and the my_ddot + MPI_Iallreduce pairs that follow them (solver.c:88-91,
// 96-102, 238-247, 365-367, 381-385).
//
//  spmv_ws_kernel<LANES, CTHREADS>   (kind 0, the default) -- warp-specialised, TMA-fed
//      Persistent CTAs walk a precomputed tile plan (<= CTHREADS/LANES rows and <= cap entries per tile).
//      One PRODUCER warp streams, per tile, everything the consumers will touch except x itself -- the val[]
//      and col[] slices, the ptr[] slice of the tile's rows and the slices of the epilogue vectors (r#, q, ...)
//      -- from HBM into a multi-stage shared-memory ring with 1-D TMA bulk copies (cp.async.bulk + mbarrier
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
//  spmv_rowsplit_kernel<LANES>       (kind 1)
//      Classic sub-warp-per-row kernel reading val/col straight from global memory; fallback for matrices
//      with rows longer than a stage, and the comparison point for the TMA kernel.
//
// Both write y exactly once (no zero-fill + accumulate passes as in matrix.c:434-440).
#include "spmv.cuh"

namespace bicg {

namespace {

__device__ __forceinline__ bool needs_tail(const KernelCommon &kc)
{
    return kc.tail.op != TAIL_NONE || kc.tail.signal_halo;
}

struct StageHdr { int row0, row1; unsigned a0; int rowa; };

template <int LANES, int CTHREADS>
__global__ void __launch_bounds__(CTHREADS + 32, 1) spmv_ws_kernel(const __grid_constant__ SpmvArgs a)
{
    if (a.kc.sc->done) return;

    constexpr int RPT = CTHREADS / LANES;            // rows per tile
    constexpr int PROW = RPT + PROW_PAD;
    constexpr int NCW = CTHREADS / 32;               // consumer warps
    constexpr int UNR = (LANES == 1) ? 16 : 8;       // gathers in flight per thread

    extern __shared__ __align__(128) unsigned char dyn_smem[];
    __shared__ __align__(8) unsigned long long full_bar[4], empty_bar[4];
    __shared__ StageHdr hdr[4];
    __shared__ double scratch[32 * 4];

    const int tid = threadIdx.x;
    const int stages = a.stages, cap = a.cap;
    // stage layout: [val cap*8][epi 4*PROW*8][col cap*4][ptr PROW*4]
    const size_t stage_bytes = (size_t)cap * 12 + (size_t)PROW * 36;
    const int my_tiles = (a.ntiles > (int)blockIdx.x) ? (a.ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const int nvec = a.epi.nvec;

    if (tid == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1u);
            mbar_init(smem_u32(&empty_bar[s]), (unsigned)NCW);
        }
        mbar_fence_init();
    }
    __syncthreads();

    double dot[4] = {0.0, 0.0, 0.0, 0.0};

    if (tid >= CTHREADS) {
        // ===================================== producer warp ==========================================
        if (tid == CTHREADS) {
            for (int i = 0; i < my_tiles; ++i) {
                const int t = (int)blockIdx.x + i * (int)gridDim.x, s = i % stages;
                const int row0 = a.tile_row[t], row1 = a.tile_row[t + 1];
                const auto [a0, cnt, rowa, cntp] = tile_window(row0, row1, a.tile_nz[t], a.tile_nz[t + 1], 3u);
                if (i >= stages) mbar_wait(smem_u32(&empty_bar[s]), (unsigned)(i / stages - 1) & 1u);
                unsigned char *st = dyn_smem + (size_t)s * stage_bytes;
                double   *sval = reinterpret_cast<double *>(st);
                double   *sepi = sval + cap;
                unsigned *scol = reinterpret_cast<unsigned *>(sepi + 4 * PROW);
                unsigned *sptr = scol + cap;
                hdr[s] = StageHdr{row0, row1, a0, rowa};
                const unsigned bar = smem_u32(&full_bar[s]);
                mbar_arrive_expect_tx(bar, cnt * 12u + (unsigned)cntp * 4u + (unsigned)(nvec * cntp) * 8u);
                if (cnt) {
                    tma_load_1d(smem_u32(sval), a.val + a0, cnt * 8u, bar);
                    tma_load_1d(smem_u32(scol), a.col + a0, cnt * 4u, bar);
                }
                tma_load_1d(smem_u32(sptr), a.ptr + rowa, (unsigned)cntp * 4u, bar);
                for (int v = 0; v < nvec; ++v)
                    tma_load_1d(smem_u32(sepi + v * PROW), a.epi.vec[v] + rowa, (unsigned)cntp * 8u, bar);
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
        const double *__restrict__ x = a.x;
        const int ndot = a.epi.ndot;

        for (int i = 0; i < my_tiles; ++i) {
            const int s = i % stages;
            mbar_wait(smem_u32(&full_bar[s]), (unsigned)(i / stages) & 1u);

            const unsigned char *st = dyn_smem + (size_t)s * stage_bytes;
            const double   *sval = reinterpret_cast<const double *>(st);
            const double   *sepi = sval + cap;
            const unsigned *scol = reinterpret_cast<const unsigned *>(sepi + 4 * PROW);
            const unsigned *sptr = scol + cap;
            const StageHdr h = hdr[s];
            const int row = h.row0 + row_in_tile;
            const bool valid = row < h.row1;
            int j = 0, e = 0;
            if (valid) {
                j = (int)(sptr[row - h.rowa] - h.a0) + lane;
                e = (int)(sptr[row - h.rowa + 1] - h.a0);
            }
            double acc = row_product<LANES, UNR>([&](int idx) { return sval[idx]; }, [&](int idx) { return scol[idx]; }, x, j, e);
            if (valid && lane == 0) {
                if (a.shift_sigma) acc = fma(*a.shift_sigma, ld_coherent(x + row), acc);     // s += sigma p (daxpy after the SpMV)
                a.y[row] = acc;
                const int ro = row - h.rowa;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (k < ndot) {
                        const double av = a.epi.ia[k] >= 0 ? sepi[a.epi.ia[k] * PROW + ro] : acc;
                        const double bv = a.epi.ib[k] >= 0 ? sepi[a.epi.ib[k] * PROW + ro] : acc;
                        dot[k] = fma(av, bv, dot[k]);
                    }
                }
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(smem_u32(&empty_bar[s]));   // this warp is done with stage s
        }
    }

    if (!needs_tail(a.kc)) return;
    block_sum<4>(dot, scratch);
    kernel_tail<4>(a.kc, dot, scratch);
}

template <int LANES>
__global__ void __launch_bounds__(256) spmv_rowsplit_kernel(const __grid_constant__ SpmvArgs a)
{
    if (a.kc.sc->done) return;
    __shared__ double scratch[32 * 4];
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
    const double *__restrict__ x = a.x;
    const double *__restrict__ val = a.val;
    const unsigned *__restrict__ col = a.col;
    const int ndot = a.epi.ndot;
    double dot[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long base = (long long)blockIdx.x * RPB; base < a.rows; base += (long long)gridDim.x * RPB) {
        const int row = (int)base + tid / LANES;
        const bool valid = row < a.rows;
        unsigned pb = 0, pe = 0;
        if (valid) { pb = a.ptr[row]; pe = a.ptr[row + 1]; }
        double acc = 0.0;
        unsigned j = pb + lane;
        for (; j + 3 * LANES < pe; j += 4 * LANES) {
            const unsigned c0 = col[j], c1 = col[j + LANES], c2 = col[j + 2 * LANES], c3 = col[j + 3 * LANES];
            const double v0 = val[j], v1 = val[j + LANES], v2 = val[j + 2 * LANES], v3 = val[j + 3 * LANES];
            acc = fma(v0, ld_coherent(x + c0), acc);
            acc = fma(v1, ld_coherent(x + c1), acc);
            acc = fma(v2, ld_coherent(x + c2), acc);
            acc = fma(v3, ld_coherent(x + c3), acc);
        }
        for (; j < pe; j += LANES) acc = fma(val[j], ld_coherent(x + col[j]), acc);
        acc = lanes_sum<LANES>(acc);
        if (valid && lane == 0) {
            if (a.shift_sigma) acc = fma(*a.shift_sigma, ld_coherent(x + row), acc);
            a.y[row] = acc;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (k < ndot) {
                    const double av = a.epi.ia[k] >= 0 ? a.epi.vec[a.epi.ia[k]][row] : acc;
                    const double bv = a.epi.ib[k] >= 0 ? a.epi.vec[a.epi.ib[k]][row] : acc;
                    dot[k] = fma(av, bv, dot[k]);
                }
            }
        }
    }
    if (!needs_tail(a.kc)) return;
    block_sum<4>(dot, scratch);
    kernel_tail<4>(a.kc, dot, scratch);
}

// ---- the batched multiply (bicg_matrix_multiply) ----------------------------------------------------------------------
// UNR * NV gathers in flight per thread: as many as the one-vector kernels keep (16 at LANES = 1, else 8)
template <int LANES, int NV>
constexpr int mul_unr() { return ((LANES == 1 ? 16 : 8) / NV) > 0 ? (LANES == 1 ? 16 : 8) / NV : 1; }

// the epilogue of row `row` for every vector of the launch: t = rowsum (+ sigma_v x_v[row]), y_v = alpha t (+ beta y_v)
template <int NV>
__device__ __forceinline__ void multiply_store(const MultiplyArgs &a, int row, const double (&acc)[NV])
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

// spmv_ws_kernel's tile walk with NV row sums per row: the producer streams val / col / ptr of a tile once for all of them
template <int LANES, int CTHREADS, int NV>
__global__ void __launch_bounds__(CTHREADS + 32, 1) multiply_ws_kernel(const __grid_constant__ MultiplyArgs a)
{
    constexpr int RPT = CTHREADS / LANES;
    constexpr int PROW = RPT + PROW_PAD;
    constexpr int NCW = CTHREADS / 32;
    constexpr int UNR = mul_unr<LANES, NV>();

    extern __shared__ __align__(128) unsigned char dyn_smem[];
    __shared__ __align__(8) unsigned long long full_bar[4], empty_bar[4];
    __shared__ StageHdr hdr[4];
    __shared__ double scratch[32];

    const int tid = threadIdx.x;
    const int stages = a.stages, cap = a.cap;
    // stage layout: [val cap*8][col cap*4][ptr PROW*4]
    const size_t stage_bytes = (size_t)cap * 12 + (size_t)PROW * 4;
    const int my_tiles = (a.ntiles > (int)blockIdx.x) ? (a.ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

    if (tid == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1u);
            mbar_init(smem_u32(&empty_bar[s]), (unsigned)NCW);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (tid >= CTHREADS) {
        if (tid == CTHREADS) {
            for (int i = 0; i < my_tiles; ++i) {
                const int t = (int)blockIdx.x + i * (int)gridDim.x, s = i % stages;
                const int row0 = a.tile_row[t], row1 = a.tile_row[t + 1];
                const auto [a0, cnt, rowa, cntp] = tile_window(row0, row1, a.tile_nz[t], a.tile_nz[t + 1], 3u);
                if (i >= stages) mbar_wait(smem_u32(&empty_bar[s]), (unsigned)(i / stages - 1) & 1u);
                unsigned char *st = dyn_smem + (size_t)s * stage_bytes;
                double   *sval = reinterpret_cast<double *>(st);
                unsigned *scol = reinterpret_cast<unsigned *>(sval + cap);
                unsigned *sptr = scol + cap;
                hdr[s] = StageHdr{row0, row1, a0, rowa};
                const unsigned bar = smem_u32(&full_bar[s]);
                mbar_arrive_expect_tx(bar, cnt * 12u + (unsigned)cntp * 4u);
                if (cnt) {
                    tma_load_1d(smem_u32(sval), a.val + a0, cnt * 8u, bar);
                    tma_load_1d(smem_u32(scol), a.col + a0, cnt * 4u, bar);
                }
                tma_load_1d(smem_u32(sptr), a.ptr + rowa, (unsigned)cntp * 4u, bar);
            }
        }
    } else {
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

        for (int i = 0; i < my_tiles; ++i) {
            const int s = i % stages;
            mbar_wait(smem_u32(&full_bar[s]), (unsigned)(i / stages) & 1u);

            const unsigned char *st = dyn_smem + (size_t)s * stage_bytes;
            const double   *sval = reinterpret_cast<const double *>(st);
            const unsigned *scol = reinterpret_cast<const unsigned *>(sval + cap);
            const unsigned *sptr = scol + cap;
            const StageHdr h = hdr[s];
            const int row = h.row0 + row_in_tile;
            const bool valid = row < h.row1;
            int j = 0, e = 0;
            if (valid) {
                j = (int)(sptr[row - h.rowa] - h.a0) + lane;
                e = (int)(sptr[row - h.rowa + 1] - h.a0);
            }
            double acc[NV];
            row_products<LANES, UNR, NV>([&](int idx) { return sval[idx]; }, [&](int idx) { return scol[idx]; }, x, j, e, acc);
            if (valid && lane == 0) multiply_store<NV>(a, row, acc);
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(smem_u32(&empty_bar[s]));
        }
    }

    if (a.kc.tail.op == TAIL_NONE) return;
    double none[1] = {0.0};
    kernel_tail<0>(a.kc, none, scratch);
}

// spmv_rowsplit_kernel's rows with NV row sums per row
template <int LANES, int NV>
__global__ void __launch_bounds__(256) multiply_rowsplit_kernel(const __grid_constant__ MultiplyArgs a)
{
    constexpr int UNR = mul_unr<LANES, NV>();
    __shared__ double scratch[32];
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
    for (long long base = (long long)blockIdx.x * RPB; base < a.rows; base += (long long)gridDim.x * RPB) {
        const int row = (int)base + tid / LANES;
        const bool valid = row < a.rows;
        unsigned pb = 0, pe = 0;
        if (valid) { pb = a.ptr[row]; pe = a.ptr[row + 1]; }
        // entries relative to the row's first one, in the order of spmv_rowsplit_kernel's loop
        const double *__restrict__ rv = a.val + pb;
        const unsigned *__restrict__ rc = a.col + pb;
        double acc[NV];
        row_products<LANES, UNR, NV>([&](int idx) { return rv[idx]; }, [&](int idx) { return rc[idx]; }, x, lane, (int)(pe - pb), acc);
        if (valid && lane == 0) multiply_store<NV>(a, row, acc);
    }
    if (a.kc.tail.op == TAIL_NONE) return;
    double none[1] = {0.0};
    kernel_tail<0>(a.kc, none, scratch);
}

template <int LANES, int CTHREADS, int NV>
cudaError_t launch_mul_ws(int grid, size_t smem, const MultiplyArgs &a, cudaStream_t st)
{
    multiply_ws_kernel<LANES, CTHREADS, NV><<<grid, CTHREADS + 32, smem, st>>>(a);
    return cudaGetLastError();
}
template <int LANES, int NV>
cudaError_t launch_mul_ws_t(int threads, int grid, size_t smem, const MultiplyArgs &a, cudaStream_t st)
{
    switch (threads) {
    case 128: return launch_mul_ws<LANES, 128, NV>(grid, smem, a, st);
    case 256: return launch_mul_ws<LANES, 256, NV>(grid, smem, a, st);
    case 512: return launch_mul_ws<LANES, 512, NV>(grid, smem, a, st);
    default:  return cudaErrorInvalidValue;
    }
}
template <int NV>
cudaError_t launch_mul_nv(int kind, int lanes, int threads, int grid, size_t smem, const MultiplyArgs &a, cudaStream_t st)
{
    if (kind == 0) {
        switch (lanes) {
        case 1:  return launch_mul_ws_t<1, NV>(threads, grid, smem, a, st);
        case 2:  return launch_mul_ws_t<2, NV>(threads, grid, smem, a, st);
        case 4:  return launch_mul_ws_t<4, NV>(threads, grid, smem, a, st);
        case 8:  return launch_mul_ws_t<8, NV>(threads, grid, smem, a, st);
        case 16: return launch_mul_ws_t<16, NV>(threads, grid, smem, a, st);
        case 32: return launch_mul_ws_t<32, NV>(threads, grid, smem, a, st);
        default: return cudaErrorInvalidValue;
        }
    }
    switch (lanes) {
    case 1:  multiply_rowsplit_kernel<1, NV><<<grid, 256, 0, st>>>(a); break;
    case 2:  multiply_rowsplit_kernel<2, NV><<<grid, 256, 0, st>>>(a); break;
    case 4:  multiply_rowsplit_kernel<4, NV><<<grid, 256, 0, st>>>(a); break;
    case 8:  multiply_rowsplit_kernel<8, NV><<<grid, 256, 0, st>>>(a); break;
    case 16: multiply_rowsplit_kernel<16, NV><<<grid, 256, 0, st>>>(a); break;
    case 32: multiply_rowsplit_kernel<32, NV><<<grid, 256, 0, st>>>(a); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

template <int LANES, int CTHREADS>
cudaError_t launch_ws(int grid, size_t smem, const SpmvArgs &a, cudaStream_t st)
{
    spmv_ws_kernel<LANES, CTHREADS><<<grid, CTHREADS + 32, smem, st>>>(a);
    return cudaGetLastError();
}
template <int LANES>
cudaError_t launch_ws_t(int threads, int grid, size_t smem, const SpmvArgs &a, cudaStream_t st)
{
    switch (threads) {
    case 128: return launch_ws<LANES, 128>(grid, smem, a, st);
    case 256: return launch_ws<LANES, 256>(grid, smem, a, st);
    case 512: return launch_ws<LANES, 512>(grid, smem, a, st);
    default:  return cudaErrorInvalidValue;
    }
}
template <int LANES>
cudaError_t launch_rowsplit(int grid, const SpmvArgs &a, cudaStream_t st)
{
    spmv_rowsplit_kernel<LANES><<<grid, 256, 0, st>>>(a);
    return cudaGetLastError();
}

template <int LANES, int CTHREADS>
cudaError_t set_attr()
{
    // opt-in limit is 227 KB per CTA *including* the kernel's static shared memory
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, spmv_ws_kernel<LANES, CTHREADS>);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(spmv_ws_kernel<LANES, CTHREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                227 * 1024 - (int)fa.sharedSizeBytes);
}
template <int LANES>
cudaError_t set_attr_l()
{
    cudaError_t e;
    if ((e = set_attr<LANES, 128>()) != cudaSuccess) return e;
    if ((e = set_attr<LANES, 256>()) != cudaSuccess) return e;
    return set_attr<LANES, 512>();
}

template <int LANES, int CTHREADS, int NV>
cudaError_t set_mul_attr()
{
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, multiply_ws_kernel<LANES, CTHREADS, NV>);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(multiply_ws_kernel<LANES, CTHREADS, NV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                227 * 1024 - (int)fa.sharedSizeBytes);
}
template <int LANES, int NV>
cudaError_t set_mul_attr_l()
{
    cudaError_t e;
    if ((e = set_mul_attr<LANES, 128, NV>()) != cudaSuccess) return e;
    if ((e = set_mul_attr<LANES, 256, NV>()) != cudaSuccess) return e;
    return set_mul_attr<LANES, 512, NV>();
}
template <int NV>
cudaError_t set_mul_attr_nv()
{
    cudaError_t e;
    if ((e = set_mul_attr_l<1, NV>()) != cudaSuccess) return e;
    if ((e = set_mul_attr_l<2, NV>()) != cudaSuccess) return e;
    if ((e = set_mul_attr_l<4, NV>()) != cudaSuccess) return e;
    if ((e = set_mul_attr_l<8, NV>()) != cudaSuccess) return e;
    if ((e = set_mul_attr_l<16, NV>()) != cudaSuccess) return e;
    return set_mul_attr_l<32, NV>();
}

} // namespace

size_t spmv_tma_smem_bytes(int cap, int stages, int threads, int lanes)
{
    const size_t prow = (size_t)(threads / lanes + PROW_PAD);
    return (size_t)stages * ((size_t)cap * 12u + prow * 36u);
}

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
    if ((e = set_attr_l<1>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_l<2>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_l<4>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_l<8>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_l<16>()) != cudaSuccess) return (int)e;
    if ((e = set_attr_l<32>()) != cudaSuccess) return (int)e;
    if ((e = set_mul_attr_nv<1>()) != cudaSuccess) return (int)e;
    if ((e = set_mul_attr_nv<2>()) != cudaSuccess) return (int)e;
    if ((e = set_mul_attr_nv<4>()) != cudaSuccess) return (int)e;
    if ((e = set_mul_attr_nv<8>()) != cudaSuccess) return (int)e;
    return 0;
}

size_t multiply_tma_smem_bytes(int cap, int stages, int threads, int lanes)
{
    const size_t prow = (size_t)(threads / lanes + PROW_PAD);
    return (size_t)stages * ((size_t)cap * 12u + prow * 4u);
}

int multiply_nv(int nv) { return nv <= 1 ? 1 : nv <= 2 ? 2 : nv <= 4 ? 4 : 8; }

int launch_multiply(int kind, int lanes, int threads, int grid, size_t smem, int NV, const MultiplyArgs &a, cudaStream_t st)
{
    switch (NV) {
    case 1:  return (int)launch_mul_nv<1>(kind, lanes, threads, grid, smem, a, st);
    case 2:  return (int)launch_mul_nv<2>(kind, lanes, threads, grid, smem, a, st);
    case 4:  return (int)launch_mul_nv<4>(kind, lanes, threads, grid, smem, a, st);
    case 8:  return (int)launch_mul_nv<8>(kind, lanes, threads, grid, smem, a, st);
    default: return (int)cudaErrorInvalidValue;
    }
}

int launch_spmv(int kind, int lanes, int threads, int grid, size_t smem, const SpmvArgs &a, cudaStream_t st)
{
    if (kind == 0) {
        switch (lanes) {
        case 1:  return (int)launch_ws_t<1>(threads, grid, smem, a, st);
        case 2:  return (int)launch_ws_t<2>(threads, grid, smem, a, st);
        case 4:  return (int)launch_ws_t<4>(threads, grid, smem, a, st);
        case 8:  return (int)launch_ws_t<8>(threads, grid, smem, a, st);
        case 16: return (int)launch_ws_t<16>(threads, grid, smem, a, st);
        case 32: return (int)launch_ws_t<32>(threads, grid, smem, a, st);
        default: return (int)cudaErrorInvalidValue;
        }
    }
    switch (lanes) {
    case 1:  return (int)launch_rowsplit<1>(grid, a, st);
    case 2:  return (int)launch_rowsplit<2>(grid, a, st);
    case 4:  return (int)launch_rowsplit<4>(grid, a, st);
    case 8:  return (int)launch_rowsplit<8>(grid, a, st);
    case 16: return (int)launch_rowsplit<16>(grid, a, st);
    case 32: return (int)launch_rowsplit<32>(grid, a, st);
    default: return (int)cudaErrorInvalidValue;
    }
}

} // namespace bicg
