// transpose.cu -- A^T of a resident matrix as a handle of its own (bicg_matrix_create_transpose), and the refresh of its values
// from the source's current values on the device (bicg_matrix_transpose_values / _async).
//
// Pattern: row j of A^T holds the entries (i, j) of A, by ascending i; entries with equal (i, j) keep their order in row i of
// A.  The transpose is built on the host from the source's merged pattern (read back from the device) by a counting sort over
// the entries taken in ascending global row, which is stable, so the order follows.  With peers, an entry (i, j) whose column
// another rank owns travels to that rank once, at creation, through the host allgather.  The blocks so built go through
// matrix_create like any caller's, so every plan of the transpose is the one a fresh handle on the same blocks gets.
//
// Refresh: every entry of the transpose's merged values is a copy of one source value.  A local one comes from the source's
// d_val through d_tperm; one whose row of A another rank owns comes from the receive region in the transpose's arena, which
// that rank fills first with a push kernel through the IPC mapping.  Then the value tables are rebuilt by the pass every value
// update runs.  Nothing here is in a solver loop.
#include "engine.hpp"

#include <algorithm>
#include <cstring>

namespace bicg {

namespace {

struct PushDst { double *recv[MAX_RANKS]; };

// the source's values that other ranks' transposes hold, into their receive regions
__global__ void __launch_bounds__(256) transpose_push_kernel(const double *__restrict__ src_val, const TransposePush *__restrict__ runs,
                                                             int n, const __grid_constant__ PushDst dst)
{
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const TransposePush p = runs[e];
        dst.recv[p.rank][p.slot] = src_val[p.src];
    }
}

// every merged value of the transpose: a local source value or a received one
__global__ void __launch_bounds__(256) transpose_gather_kernel(const double *__restrict__ src_val, const double *__restrict__ recv,
                                                               const int *__restrict__ perm, size_t n, double *__restrict__ val)
{
    for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
        const int s = perm[k];
        val[k] = s >= 0 ? src_val[s] : recv[~s];
    }
}

int grid_for(size_t n) { return (int)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)ctx().sm_count * 8)); }

// the refresh on st, behind both handles' earlier work (the caller has made st wait for it)
void enqueue_refresh(bicg_matrix *mt, const bicg_matrix *src, cudaStream_t st)
{
    if (mt->world > 1) {
        // nobody stores into a receive region its owner has not consumed yet; then every push has landed
        BICG_CUDA(cudaMemsetAsync(&mt->d_sc->done, 0, sizeof(int), st));
        peer_barrier(mt, st);
        if (mt->t_npush) {
            PushDst dst{};
            for (int p = 0; p < mt->world; ++p) dst.recv[p] = mt->peer_trecv[p];
            transpose_push_kernel<<<grid_for((size_t)mt->t_npush), 256, 0, st>>>(src->d_val, mt->d_tpush, mt->t_npush, dst);
            BICG_CUDA(cudaGetLastError());
        }
        peer_barrier(mt, st);
    }
    if (mt->nnz) {
        transpose_gather_kernel<<<grid_for(mt->nnz), 256, 0, st>>>(src->d_val, mt->d_trecv, mt->d_tperm, mt->nnz, mt->d_val);
        BICG_CUDA(cudaGetLastError());
    }
    launch_value_tables(mt, st);
}

// the -1 case of both refresh calls: mt is not a transpose of src
bool transpose_bad(const bicg_matrix *mt, const bicg_matrix *src)
{
    return !mt || !src || !mt->t_src_uid || mt->t_src_uid != src->uid;
}

template <class T> void d2h(std::vector<T> &out, const T *d, size_t n)
{
    out.resize(n);
    if (n) BICG_CUDA(cudaMemcpy(out.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost));
}

// one source entry of a row of the transpose: its column there (the global row of A) and where its value comes from
struct TEntry { unsigned gi; int src; };

} // namespace

} // namespace bicg

extern "C" bicg_matrix *bicg_matrix_create_transpose(bicg_matrix *m)
{
    using namespace bicg;
    Context &c = ctx();
    // collective: every rank learns whether any rank passed a null handle, and every rank's row count (the partition of m)
    struct Mine { int ok, n_loc; } mine{m ? 1 : 0, m ? m->n_loc : 0};
    std::vector<Mine> all((size_t)c.world);
    c.host_allgather(&mine, all.data(), sizeof(Mine));
    for (const Mine &o : all) if (!o.ok) return nullptr;
    c.ensure();
    wait_handle(m);
    BICG_CUDA(cudaStreamSynchronize(c.stream));
    const int W = m->world, me = m->rank, n_loc = m->n_loc;
    std::vector<int> cnt((size_t)W), dsp((size_t)W + 1, 0);
    for (int p = 0; p < W; ++p) { cnt[(size_t)p] = all[(size_t)p].n_loc; dsp[(size_t)p + 1] = dsp[(size_t)p] + cnt[(size_t)p]; }
    const unsigned lo = (unsigned)dsp[(size_t)me];
    auto owner = [&](unsigned g) { return (int)(std::upper_bound(dsp.begin() + 1, dsp.end(), (int)g) - (dsp.begin() + 1)); };

    // ---- the source's pattern: global row and column of every merged entry ----------------------------------------------
    std::vector<unsigned> ptr, col;
    d2h(ptr, m->d_ptr, (size_t)n_loc + 1);
    d2h(col, m->d_col, m->nnz);
    std::vector<unsigned> ghost_gc((size_t)m->n_ghost);          // ghost slot -> global column
    for (size_t r = 0; r + 3 < m->recv_runs.size(); r += 4)
        for (int t = 0; t < m->recv_runs[r + 1]; ++t) ghost_gc[(size_t)(m->recv_runs[r + 3] + t)] = (unsigned)(m->recv_runs[r] + t);
    auto gcol = [&](size_t k) { return col[k] < (unsigned)m->ghost_off ? lo + col[k] : ghost_gc[col[k] - (unsigned)m->ghost_off]; };

    // ---- entries whose column another rank owns go to that rank: (global row, global column), by ascending entry ---------
    std::vector<int> send_cnt((size_t)W, 0);
    for (int i = 0; i < n_loc; ++i)
        for (unsigned k = ptr[(size_t)i]; k < ptr[(size_t)i + 1]; ++k) {
            const int p = owner(gcol(k));
            if (p != me) ++send_cnt[(size_t)p];
        }
    std::vector<int> cnt_all((size_t)W * W);                      // cnt_all[q * W + p]: entries q sends to p
    c.host_allgather(send_cnt.data(), cnt_all.data(), (size_t)W * sizeof(int));
    size_t max_send = 1;
    for (int q = 0; q < W; ++q) {
        size_t s = 0;
        for (int p = 0; p < W; ++p) s += (size_t)cnt_all[(size_t)q * W + p];
        max_send = std::max(max_send, s);
    }
    // slot of q's e-th entry for p in p's receive region: the entries of lower ranks first
    auto slot_base = [&](int q, int p) { int b = 0; for (int r = 0; r < q; ++r) b += cnt_all[(size_t)r * W + p]; return b; };
    std::vector<size_t> send_off((size_t)W + 1, 0);
    for (int p = 0; p < W; ++p) send_off[(size_t)p + 1] = send_off[(size_t)p] + (size_t)send_cnt[(size_t)p];
    std::vector<unsigned> send(2 * max_send, 0);
    std::vector<TransposePush> push;
    push.reserve(send_off[(size_t)W]);
    {
        std::vector<size_t> fill(send_off.begin(), send_off.end() - 1);
        for (int i = 0; i < n_loc; ++i)
            for (unsigned k = ptr[(size_t)i]; k < ptr[(size_t)i + 1]; ++k) {
                const unsigned g = gcol(k);
                const int p = owner(g);
                if (p == me) continue;
                const size_t e = fill[(size_t)p]++;
                send[2 * e] = lo + (unsigned)i; send[2 * e + 1] = g;
                push.push_back(TransposePush{(int)k, p, slot_base(me, p) + (int)(e - send_off[(size_t)p])});
            }
    }
    std::vector<unsigned> recv;
    if (W > 1) {
        recv.resize(2 * max_send * (size_t)W);
        c.host_allgather(send.data(), recv.data(), 2 * max_send * sizeof(unsigned));
    }

    // ---- rows of the transpose: a counting sort over the entries in ascending global row of A, rank by rank --------------
    // (the source rank's own entries ascend in row and, within a row, in merged order; so do the ones q sent)
    std::vector<size_t> rp((size_t)n_loc + 1, 0);
    auto for_each_entry = [&](auto &&visit) {                    // visit(row of A^T, TEntry)
        size_t nrecv = 0;
        for (int q = 0; q < W; ++q) {
            if (q == me) {
                for (int i = 0; i < n_loc; ++i)
                    for (unsigned k = ptr[(size_t)i]; k < ptr[(size_t)i + 1]; ++k) {
                        const unsigned g = gcol(k);
                        if (g >= lo && g < lo + (unsigned)n_loc) visit(g - lo, TEntry{lo + (unsigned)i, (int)k});
                    }
                continue;
            }
            // q's entries for me sit behind those it sent to lower ranks
            size_t off = 0;
            for (int p = 0; p < me; ++p) off += (size_t)cnt_all[(size_t)q * W + p];
            const unsigned *src = recv.data() + 2 * (max_send * (size_t)q + off);
            for (int e = 0; e < cnt_all[(size_t)q * W + me]; ++e, ++nrecv)
                visit(src[2 * e + 1] - lo, TEntry{src[2 * e], ~(int)nrecv});
        }
        return nrecv;
    };
    const size_t nrecv = for_each_entry([&](unsigned j, TEntry) { ++rp[(size_t)j + 1]; });
    for (int j = 0; j < n_loc; ++j) rp[(size_t)j + 1] += rp[(size_t)j];
    std::vector<TEntry> ent(rp[(size_t)n_loc]);
    {
        std::vector<size_t> fill(rp.begin(), rp.end() - 1);
        for_each_entry([&](unsigned j, TEntry t) { ent[fill[j]++] = t; });
    }

    // ---- the transpose's blocks (diag: own columns, local; offd: global), and the source of every merged entry ------------
    std::vector<unsigned> dptr((size_t)n_loc + 1, 0), optr((size_t)n_loc + 1, 0), dcol, ocol;
    std::vector<int> perm;
    perm.reserve(ent.size());
    dcol.reserve(ent.size());
    for (int j = 0; j < n_loc; ++j) {
        for (size_t e = rp[(size_t)j]; e < rp[(size_t)j + 1]; ++e)          // the merged row: diag entries first ...
            if (ent[e].gi >= lo && ent[e].gi < lo + (unsigned)n_loc) { dcol.push_back(ent[e].gi - lo); perm.push_back(ent[e].src); }
        for (size_t e = rp[(size_t)j]; e < rp[(size_t)j + 1]; ++e)          // ... then offd entries
            if (!(ent[e].gi >= lo && ent[e].gi < lo + (unsigned)n_loc)) { ocol.push_back(ent[e].gi); perm.push_back(ent[e].src); }
        dptr[(size_t)j + 1] = (unsigned)dcol.size();
        optr[(size_t)j + 1] = (unsigned)ocol.size();
    }
    std::vector<double> dval(std::max<size_t>(dcol.size(), 1), 0.0), oval(std::max<size_t>(ocol.size(), 1), 0.0);
    if (dcol.empty()) dcol.push_back(0);
    if (ocol.empty()) ocol.push_back(0);
    CSR_Matrix D{dval.data(), dcol.data(), dptr.data(), dptr[(size_t)n_loc], (unsigned)n_loc, (unsigned)n_loc};
    CSR_Matrix O{oval.data(), ocol.data(), optr.data(), optr[(size_t)n_loc], (unsigned)n_loc, (unsigned)m->n_glob};
    std::vector<int> recvcounts(cnt), displs(dsp.begin(), dsp.end() - 1);
    unsigned long long nz_mine = m->nnz;
    std::vector<unsigned long long> nz_all((size_t)W);
    c.host_allgather(&nz_mine, nz_all.data(), sizeof(nz_mine));
    unsigned long long nz = 0;
    for (unsigned long long v : nz_all) nz += v;
    INFO_Matrix info{};
    info.nz = (unsigned)nz; info.rows = (unsigned)m->n_glob; info.cols = (unsigned)m->n_glob;
    memcpy(info.code, "MCRG", 4);
    info.recvcounts = recvcounts.data(); info.displs = displs.data();

    bicg_matrix *mt = matrix_create(&D, &O, &info, nrecv);
    mt->t_src_uid = m->uid;
    if (!perm.empty()) {
        mt->d_tperm = (int *)c.dev_alloc(perm.size() * sizeof(int));
        BICG_CUDA(cudaMemcpyAsync(mt->d_tperm, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
    }
    mt->t_npush = (int)push.size();
    if (!push.empty()) {
        mt->d_tpush = (TransposePush *)c.dev_alloc(push.size() * sizeof(TransposePush));
        BICG_CUDA(cudaMemcpyAsync(mt->d_tpush, push.data(), push.size() * sizeof(TransposePush), cudaMemcpyHostToDevice, c.stream));
    }
    // the values: the refresh every later bicg_matrix_transpose_values runs
    enqueue_refresh(mt, m, c.stream);
    sync_checked(mt, "the creation of a transpose");
    return mt;
}

extern "C" int bicg_matrix_transpose_values(bicg_matrix *mt, bicg_matrix *src)
{
    using namespace bicg;
    Context &c = ctx();
    // collective (the barriers of the refresh): every rank's verdict
    if (!ranks_agree(transpose_bad(mt, src), {})) return -1;
    c.ensure();
    wait_handle(mt);
    wait_handle(src);
    enqueue_refresh(mt, src, c.stream);
    sync_checked(mt, "a transpose refresh");
    return 0;
}

extern "C" int bicg_matrix_transpose_values_async(bicg_matrix *mt, bicg_matrix *src, void *stream)
{
    using namespace bicg;
    if (transpose_bad(mt, src)) return -1;
    ctx().ensure();
    const cudaStream_t st = (cudaStream_t)stream;
    stream_ordered({mt, src}, st, capturing(st), [&] { enqueue_refresh(mt, src, st); });
    return 0;
}
