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
//
// Entry permutation (bicg_matrix_transpose_entries_async): the refresh's copies on caller vectors in the block orders
// set_values takes, forward (source -> transpose) through the same push and gather over block-order tables, and reverse
// through the opposite traffic: every transposed entry that came from another rank goes back into a second region of that
// rank's receive area, from which it is scattered to its source position.  All tables are built here at creation.
#include "engine.hpp"

#include <algorithm>
#include <cstring>

namespace bicg {

namespace {

struct PushDst { double *recv[MAX_RANKS]; };

// an entry vector read by index: merged values (diag = d_val, nd = nnz), or the two blocks set_values takes (index b < nd is
// diag entry b, else offd entry b - nd)
struct Entries {
    const double *diag, *offd;
    size_t nd;
    __device__ __forceinline__ double operator[](size_t b) const { return b < nd ? diag[b] : offd[b - nd]; }
};
struct OutEntries {
    double *diag, *offd;
    size_t nd;
    __device__ __forceinline__ double &operator[](size_t b) const { return b < nd ? diag[b] : offd[b - nd]; }
};

// the entries of `in` that other ranks hold, into their receive regions
__global__ void __launch_bounds__(256) transpose_push_kernel(const Entries in, const TransposePush *__restrict__ runs, int n,
                                                             const __grid_constant__ PushDst dst)
{
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const TransposePush p = runs[e];
        dst.recv[p.rank][p.slot] = in[(size_t)p.src];
    }
}

// every entry of the transpose: a local source entry or a received one
__global__ void __launch_bounds__(256) transpose_gather_kernel(const Entries in, const double *__restrict__ recv,
                                                               const int *__restrict__ perm, size_t n, const OutEntries out)
{
    for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
        const int s = perm[k];
        out[k] = s >= 0 ? in[(size_t)s] : recv[~s];
    }
}

// the inverse of a gather over the entries with perm[k] >= 0: out[perm[k]] = in[k]
__global__ void __launch_bounds__(256) transpose_scatter_kernel(const Entries in, const int *__restrict__ perm, size_t n,
                                                                const OutEntries out)
{
    for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
        const int s = perm[k];
        if (s >= 0) out[(size_t)s] = in[k];
    }
}

int grid_for(size_t n) { return (int)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)ctx().sm_count * 8)); }

PushDst push_dst(const bicg_matrix *mt)
{
    PushDst dst{};
    for (int p = 0; p < mt->world; ++p) dst.recv[p] = mt->peer_trecv[p];
    return dst;
}

// with peers: `runs` (n of them) store entries of `in` into the receive regions of mt's peers, between two empty cross-GPU
// reductions: nobody stores into a receive region its owner has not consumed yet, and then every push has landed
void exchange(bicg_matrix *mt, const Entries &in, const TransposePush *runs, int n, cudaStream_t st)
{
    BICG_CUDA(cudaMemsetAsync(&mt->d_sc->done, 0, sizeof(int), st));
    peer_barrier(mt, st);
    if (n) {
        transpose_push_kernel<<<grid_for((size_t)n), 256, 0, st>>>(in, runs, n, push_dst(mt));
        BICG_CUDA(cudaGetLastError());
    }
    peer_barrier(mt, st);
}

// the refresh on st, behind both handles' earlier work (the caller has made st wait for it)
void enqueue_refresh(bicg_matrix *mt, const bicg_matrix *src, cudaStream_t st)
{
    const Entries in{src->d_val, nullptr, src->nnz};
    if (mt->world > 1) exchange(mt, in, mt->d_tpush, mt->t_npush, st);
    if (mt->nnz) {
        transpose_gather_kernel<<<grid_for(mt->nnz), 256, 0, st>>>(in, mt->d_trecv, mt->d_tperm, mt->nnz,
                                                                  OutEntries{mt->d_val, nullptr, mt->nnz});
        BICG_CUDA(cudaGetLastError());
    }
    launch_value_tables(mt, st);
}

// bicg_matrix_transpose_entries_async on st: forward, src's block order -> mt's, the refresh's traffic on entry vectors; reverse,
// mt's block order -> src's, every entry back where the forward took it from
void enqueue_entries(bicg_matrix *mt, const bicg_matrix *src, int reverse, const double *in_diag, const double *in_offd,
                     double *out_diag, double *out_offd, cudaStream_t st)
{
    const size_t snd = src->nnz - src->nnz_offd, tnd = mt->nnz - mt->nnz_offd;
    if (!reverse) {
        const Entries in{in_diag, in_offd, snd};
        if (mt->world > 1) exchange(mt, in, mt->d_tbpush, mt->t_npush, st);
        if (mt->nnz) {
            transpose_gather_kernel<<<grid_for(mt->nnz), 256, 0, st>>>(in, mt->d_trecv, mt->d_tbperm, mt->nnz,
                                                                      OutEntries{out_diag, out_offd, tnd});
            BICG_CUDA(cudaGetLastError());
        }
        return;
    }
    const Entries in{in_diag, in_offd, tnd};
    const OutEntries out{out_diag, out_offd, snd};
    if (mt->world > 1) exchange(mt, in, mt->d_trpush, mt->t_nrpush, st);
    if (mt->nnz) {
        transpose_scatter_kernel<<<grid_for(mt->nnz), 256, 0, st>>>(in, mt->d_tbperm, mt->nnz, out);
        BICG_CUDA(cudaGetLastError());
    }
    if (mt->t_npush) {
        const Entries back{mt->d_trecv + mt->t_rev_off, nullptr, (size_t)mt->t_npush};
        transpose_scatter_kernel<<<grid_for((size_t)mt->t_npush), 256, 0, st>>>(back, mt->d_trev_src, (size_t)mt->t_npush, out);
        BICG_CUDA(cudaGetLastError());
    }
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
    std::vector<int> rev_src(send_off[(size_t)W]);               // reverse region entry e (grouped by peer): source merged entry
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
                rev_src[e] = (int)k;
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

    // the receive region holds the forward entries (nrecv), then the reverse region: the entries this rank pushes forward
    bicg_matrix *mt = matrix_create(&D, &O, &info, nrecv + push.size());
    mt->t_src_uid = m->uid;
    mt->t_rev_off = nrecv;

    // ---- the tables over block orders (bicg_matrix_transpose_entries_async) ---------------------------------------------
    // merged entry -> block index, on either handle: row i's diag entries, then its offd entries (dev.cuh: merge_row)
    auto block_index = [&](const std::vector<unsigned> &bp, int rows) {
        std::vector<int> b;
        if (bp.empty()) return b;                                   // no offd entries: the orders agree
        const unsigned *bd = bp.data(), *bo = bp.data() + rows + 1;
        const int nd = (int)bd[rows];
        b.reserve((size_t)nd + bo[rows]);
        for (int i = 0; i < rows; ++i) {
            for (unsigned j = bd[i]; j < bd[i + 1]; ++j) b.push_back((int)j);
            for (unsigned j = bo[i]; j < bo[i + 1]; ++j) b.push_back(nd + (int)j);
        }
        return b;
    };
    std::vector<unsigned> sbp, tbp;
    if (m->nnz_offd) d2h(sbp, m->d_blk_ptr, 2 * ((size_t)n_loc + 1));
    if (mt->nnz_offd) {
        tbp.assign(dptr.begin(), dptr.end());
        tbp.insert(tbp.end(), optr.begin(), optr.end());
    }
    const std::vector<int> sblk = block_index(sbp, n_loc), tblk = block_index(tbp, n_loc);
    auto sb = [&](int k) { return sblk.empty() ? k : sblk[(size_t)k]; };
    auto tb = [&](size_t k) { return tblk.empty() ? k : (size_t)tblk[k]; };
    std::vector<int> bperm(perm.size());
    for (size_t k = 0; k < perm.size(); ++k) bperm[tb(k)] = perm[k] >= 0 ? sb(perm[k]) : perm[k];
    std::vector<TransposePush> bpush(push);
    for (TransposePush &p : bpush) p.src = sb(p.src);
    for (int &k : rev_src) k = sb(k);
    // every received entry goes back to the rank q that pushed it: slot s of my region is q's t-th entry for me, which sits at
    // t_rev_off(q) + (q's entries for lower ranks) + t in q's receive region
    std::vector<TransposePush> rpush;
    for (size_t k = 0; k < perm.size(); ++k) {
        if (perm[k] >= 0) continue;
        int s = ~perm[k], q = 0;
        while (s >= cnt_all[(size_t)q * W + me]) s -= cnt_all[(size_t)q++ * W + me];
        int base = 0;
        for (int r = 0; r < W; ++r) base += cnt_all[(size_t)r * W + q];            // q's nrecv
        for (int r = 0; r < me; ++r) base += cnt_all[(size_t)q * W + r];
        rpush.push_back(TransposePush{(int)tb(k), q, base + s});
    }
    if (!perm.empty()) {
        mt->d_tperm = (int *)c.dev_alloc(perm.size() * sizeof(int));
        BICG_CUDA(cudaMemcpyAsync(mt->d_tperm, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
    }
    mt->t_npush = (int)push.size();
    if (!push.empty()) {
        mt->d_tpush = (TransposePush *)c.dev_alloc(push.size() * sizeof(TransposePush));
        BICG_CUDA(cudaMemcpyAsync(mt->d_tpush, push.data(), push.size() * sizeof(TransposePush), cudaMemcpyHostToDevice, c.stream));
    }
    auto upload = [&](auto &v, auto *alias) {
        using T = typename std::decay_t<decltype(v)>::value_type;
        if (v.empty()) return (T *)nullptr;
        if (alias && std::equal(v.begin(), v.end(), alias, [](const T &a, const T &b) { return !memcmp(&a, &b, sizeof(T)); }))
            return (T *)nullptr;
        T *d = (T *)c.dev_alloc(v.size() * sizeof(T));
        BICG_CUDA(cudaMemcpyAsync(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, c.stream));
        return d;
    };
    mt->d_tbperm = upload(bperm, perm.data());
    if (!mt->d_tbperm) mt->d_tbperm = mt->d_tperm;
    mt->d_tbpush = upload(bpush, push.data());
    if (!mt->d_tbpush) mt->d_tbpush = mt->d_tpush;
    mt->d_trpush = upload(rpush, (const TransposePush *)nullptr);
    mt->t_nrpush = (int)rpush.size();
    mt->d_trev_src = upload(rev_src, (const int *)nullptr);
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

extern "C" int bicg_matrix_transpose_entries_async(bicg_matrix *mt, bicg_matrix *src, int reverse, const double *in_diag,
                                                   const double *in_offd, double *out_diag, double *out_offd, void *stream)
{
    using namespace bicg;
    if (!mt || !src || (reverse != 0 && reverse != 1) || !in_diag || !out_diag) return -1;
    const bicg_matrix *a = reverse ? mt : src, *b = reverse ? src : mt;         // in's handle, out's handle
    const size_t ano = a->nnz_offd, and_ = a->nnz - ano, bno = b->nnz_offd, bnd = b->nnz - bno;
    if ((ano && !in_offd) || (bno && !out_offd)) return -1;
    auto hits_in = [&](const void *o, size_t n) {
        return overlaps(o, n * sizeof(double), in_diag, and_ * sizeof(double)) ||
               (ano && overlaps(o, n * sizeof(double), in_offd, ano * sizeof(double)));
    };
    if (hits_in(out_diag, bnd) || (bno && hits_in(out_offd, bno)) || transpose_bad(mt, src)) return -1;
    ctx().ensure();
    const cudaStream_t st = (cudaStream_t)stream;
    stream_ordered({mt, src}, st, capturing(st),
                   [&] { enqueue_entries(mt, src, reverse, in_diag, in_offd, out_diag, out_offd, st); });
    return 0;
}
