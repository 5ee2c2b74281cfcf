// vec_body.cuh -- the element-wise bodies of the fused BLAS-1 phases, shared by the stand-alone phase kernels
// (vec.cu) and the persistent solver kernel (mega.cu).  See vec.cu for the reference lines each phase replaces.
#pragma once
#include "vec.cuh"

namespace bicg {

template <int W> struct Pk { double v[W]; };

// the accesses of one L2 policy (dev.cuh: Plain, Hint); every phase kernel of vec.cu uses Plain
__device__ __forceinline__ double ld1(const double *p, Plain) { return *p; }
__device__ __forceinline__ double ld1(const double *p, Hint h) { return ld_hint(p, h.pol); }
__device__ __forceinline__ double2 ld2(const double *p, Plain) { return *reinterpret_cast<const double2 *>(p); }
__device__ __forceinline__ double2 ld2(const double *p, Hint h) { return ld_hint2(p, h.pol); }
__device__ __forceinline__ void st1(double *p, double v, Plain) { *p = v; }
__device__ __forceinline__ void st1(double *p, double v, Hint h) { st_hint(p, v, h.pol); }
__device__ __forceinline__ void st2(double *p, double2 v, Plain) { *reinterpret_cast<double2 *>(p) = v; }
__device__ __forceinline__ void st2(double *p, double2 v, Hint h) { st_hint2(p, v, h.pol); }

// W contiguous doubles: one 8-byte access for W = 1, 16-byte accesses otherwise
template <int W, class H> __device__ __forceinline__ Pk<W> ld(const double *p, int i, H h)
{
    Pk<W> r;
    if constexpr (W == 1) {
        r.v[0] = ld1(p + i, h);
    } else {
#pragma unroll
        for (int k = 0; k < W; k += 2) { const double2 t = ld2(p + i + k, h); r.v[k] = t.x; r.v[k + 1] = t.y; }
    }
    return r;
}
template <int W, class H> __device__ __forceinline__ void st(double *p, int i, const Pk<W> &a, H h)
{
    if constexpr (W == 1) {
        st1(p + i, a.v[0], h);
    } else {
#pragma unroll
        for (int k = 0; k < W; k += 2) st2(p + i + k, make_double2(a.v[k], a.v[k + 1]), h);
    }
}

__host__ __device__ constexpr int phase_ndot(int ph)
{
    return ph == PH_BICG_INIT ? 1 : ph == PH_BICG_XR ? 2 : ph == PH_INIT_R ? 1 : ph == PH_QY ? 2
         : ph == PH_CA_XR ? 1 : ph == PH_PIPE_1 ? 2 : ph == PH_PIPE_3 ? 5 : ph == PH_RR_DOTS ? 5 : 0;
}


// access policies: W contiguous doubles (vector loads), or W doubles STRIDE apart (one per step of a
// thread-strided loop, so W independent loads are in flight per vector); each access takes the L2 policy h
template <int W_> struct Contig {
    static constexpr int W = W_;
    template <class H = Plain>
    static __device__ __forceinline__ Pk<W_> ld(const double *p, int i, H h = {}) { return bicg::ld<W_>(p, i, h); }
    template <class H = Plain>
    static __device__ __forceinline__ void st(double *p, int i, const Pk<W_> &a, H h = {}) { bicg::st<W_>(p, i, a, h); }
};
template <int W_, int STRIDE> struct Strided {
    static constexpr int W = W_;
    template <class H = Plain>
    static __device__ __forceinline__ Pk<W_> ld(const double *p, int i, H h = {})
    {
        Pk<W_> r;
#pragma unroll
        for (int k = 0; k < W_; ++k) r.v[k] = ld1(p + i + k * STRIDE, h);
        return r;
    }
    template <class H = Plain>
    static __device__ __forceinline__ void st(double *p, int i, const Pk<W_> &a, H h = {})
    {
#pragma unroll
        for (int k = 0; k < W_; ++k) st1(p + i + k * STRIDE, a.v[k], h);
    }
};

// K double2 accesses STRIDE doubles apart (persistent kernel: K independent 16-byte loads in flight per vector)
template <int K, int STRIDE> struct Pairs {
    static constexpr int W = 2 * K;
    template <class H = Plain>
    static __device__ __forceinline__ Pk<W> ld(const double *p, int i, H h = {})
    {
        Pk<W> r;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const double2 t = ld2(p + i + k * STRIDE, h);
            r.v[2 * k] = t.x; r.v[2 * k + 1] = t.y;
        }
        return r;
    }
    template <class H = Plain>
    static __device__ __forceinline__ void st(double *p, int i, const Pk<W> &a, H h = {})
    {
#pragma unroll
        for (int k = 0; k < K; ++k) st2(p + i + k * STRIDE, make_double2(a.v[2 * k], a.v[2 * k + 1]), h);
    }
};

struct Coef { double al, be, om, nbo; };

// far: the L2 policy of the accesses of PH_BICG_XR and PH_BICG_P whose next use is too far away for L2 to keep the vector
// (mega.cu: run_bicgstab's table); every other access is plain
template <int PH, class L, class F = Plain>
__device__ __forceinline__ void body(const VecPtrs &v, int i, const Coef &c, double *dot, F far = {})
{
    constexpr int W = L::W;
    if constexpr (PH == PH_BICG_INIT || PH == PH_INIT_R) {
        Pk<W> ax = L::ld(v.ax, i), r = L::ld(v.r, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            r.v[k] = fma(-1.0, ax.v[k], r.v[k]);
            dot[0] = fma(r.v[k], r.v[k], dot[0]);
        }
        L::st(v.r, i, r); L::st(v.rh, i, r);
        if constexpr (PH == PH_BICG_INIT) L::st(v.p, i, r);
    } else if constexpr (PH == PH_BICG_Q) {
        Pk<W> s = L::ld(v.s, i), r = L::ld(v.r, i);
#pragma unroll
        for (int k = 0; k < W; ++k) r.v[k] = fma(-c.al, s.v[k], r.v[k]);
        L::st(v.r, i, r);
    } else if constexpr (PH == PH_BICG_XR) {
        Pk<W> x = L::ld(v.x, i, far), p = L::ld(v.p, i), r = L::ld(v.r, i), y = L::ld(v.y, i, far), rh = L::ld(v.rh, i, far);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            x.v[k] = fma(c.al, p.v[k], x.v[k]);
            x.v[k] = fma(c.om, r.v[k], x.v[k]);
            r.v[k] = fma(-c.om, y.v[k], r.v[k]);
            dot[0] = fma(r.v[k], r.v[k], dot[0]);
            dot[1] = fma(rh.v[k], r.v[k], dot[1]);
        }
        L::st(v.x, i, x, far); L::st(v.r, i, r);
    } else if constexpr (PH == PH_BICG_P) {
        Pk<W> p = L::ld(v.p, i), r = L::ld(v.r, i), s = L::ld(v.s, i, far);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            double t = c.be * p.v[k];
            t = fma(1.0, r.v[k], t);
            p.v[k] = fma(c.nbo, s.v[k], t);
        }
        L::st(v.p, i, p);
    } else if constexpr (PH == PH_CA_PS) {
        Pk<W> p = L::ld(v.p, i), s = L::ld(v.s, i), z = L::ld(v.z, i), r = L::ld(v.r, i), w = L::ld(v.w, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            double t = fma(-c.om, s.v[k], p.v[k]);
            t = c.be * t;
            p.v[k] = fma(1.0, r.v[k], t);
            double u = fma(-c.om, z.v[k], s.v[k]);
            u = c.be * u;
            s.v[k] = fma(1.0, w.v[k], u);
        }
        L::st(v.p, i, p); L::st(v.s, i, s);
    } else if constexpr (PH == PH_QY) {
        Pk<W> r = L::ld(v.r, i), s = L::ld(v.s, i), w = L::ld(v.w, i), z = L::ld(v.z, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            r.v[k] = fma(-c.al, s.v[k], r.v[k]);
            w.v[k] = fma(-c.al, z.v[k], w.v[k]);
            dot[0] = fma(r.v[k], w.v[k], dot[0]);
            dot[1] = fma(w.v[k], w.v[k], dot[1]);
        }
        L::st(v.r, i, r); L::st(v.w, i, w);
    } else if constexpr (PH == PH_CA_XR) {
        Pk<W> x = L::ld(v.x, i), p = L::ld(v.p, i), r = L::ld(v.r, i), w = L::ld(v.w, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            x.v[k] = fma(c.al, p.v[k], x.v[k]);
            x.v[k] = fma(c.om, r.v[k], x.v[k]);
            r.v[k] = fma(-c.om, w.v[k], r.v[k]);
            dot[0] = fma(r.v[k], r.v[k], dot[0]);
        }
        L::st(v.x, i, x); L::st(v.r, i, r);
    } else if constexpr (PH == PH_PIPE_1) {
        Pk<W> p = L::ld(v.p, i), s = L::ld(v.s, i), z = L::ld(v.z, i), vv = L::ld(v.v, i), t = L::ld(v.t, i),
              r = L::ld(v.r, i), w = L::ld(v.w, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            double a = fma(-c.om, s.v[k], p.v[k]);  a = c.be * a;  p.v[k] = fma(1.0, r.v[k], a);
            double b = fma(-c.om, z.v[k], s.v[k]);  b = c.be * b;  s.v[k] = fma(1.0, w.v[k], b);
            double d = fma(-c.om, vv.v[k], z.v[k]); d = c.be * d;  z.v[k] = fma(1.0, t.v[k], d);
            r.v[k] = fma(-c.al, s.v[k], r.v[k]);
            w.v[k] = fma(-c.al, z.v[k], w.v[k]);
            dot[0] = fma(r.v[k], w.v[k], dot[0]);
            dot[1] = fma(w.v[k], w.v[k], dot[1]);
        }
        L::st(v.p, i, p); L::st(v.s, i, s); L::st(v.z, i, z); L::st(v.r, i, r); L::st(v.w, i, w);
    } else if constexpr (PH == PH_PIPE_3) {
        Pk<W> x = L::ld(v.x, i), p = L::ld(v.p, i), r = L::ld(v.r, i), w = L::ld(v.w, i), t = L::ld(v.t, i),
              vv = L::ld(v.v, i), rh = L::ld(v.rh, i), s = L::ld(v.s, i), z = L::ld(v.z, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            x.v[k] = fma(c.al, p.v[k], x.v[k]);
            x.v[k] = fma(c.om, r.v[k], x.v[k]);
            r.v[k] = fma(-c.om, w.v[k], r.v[k]);
            const double tt = fma(-c.al, vv.v[k], t.v[k]);     // t - alpha v; t itself is overwritten by t = A w next
            w.v[k] = fma(-c.om, tt, w.v[k]);
            dot[0] = fma(rh.v[k], r.v[k], dot[0]);     // order expected by FIN_CAPIPE_END
            dot[1] = fma(rh.v[k], w.v[k], dot[1]);
            dot[2] = fma(rh.v[k], s.v[k], dot[2]);
            dot[3] = fma(rh.v[k], z.v[k], dot[3]);
            dot[4] = fma(r.v[k], r.v[k], dot[4]);
        }
        L::st(v.x, i, x); L::st(v.r, i, r); L::st(v.w, i, w);
    } else if constexpr (PH == PH_RR_P) {
        Pk<W> p = L::ld(v.p, i), s = L::ld(v.s, i), r = L::ld(v.r, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            double a = fma(-c.om, s.v[k], p.v[k]); a = c.be * a; p.v[k] = fma(1.0, r.v[k], a);
        }
        L::st(v.p, i, p);
    } else if constexpr (PH == PH_RR_X) {
        Pk<W> x = L::ld(v.x, i), p = L::ld(v.p, i), r = L::ld(v.r, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            x.v[k] = fma(c.al, p.v[k], x.v[k]);
            x.v[k] = fma(c.om, r.v[k], x.v[k]);
        }
        L::st(v.x, i, x);
    } else if constexpr (PH == PH_RR_R) {
        Pk<W> b = L::ld(v.b, i), ax = L::ld(v.ax, i);
#pragma unroll
        for (int k = 0; k < W; ++k) b.v[k] = fma(-1.0, ax.v[k], b.v[k]);
        L::st(v.r, i, b);
    } else if constexpr (PH == PH_RR_DOTS) {
        Pk<W> r = L::ld(v.r, i), rh = L::ld(v.rh, i), w = L::ld(v.w, i), s = L::ld(v.s, i), z = L::ld(v.z, i);
#pragma unroll
        for (int k = 0; k < W; ++k) {
            dot[0] = fma(rh.v[k], r.v[k], dot[0]);     // order expected by FIN_CAPIPE_END
            dot[1] = fma(rh.v[k], w.v[k], dot[1]);
            dot[2] = fma(rh.v[k], s.v[k], dot[2]);
            dot[3] = fma(rh.v[k], z.v[k], dot[3]);
            dot[4] = fma(r.v[k], r.v[k], dot[4]);
        }
    }
    (void)v; (void)i; (void)c; (void)dot; (void)far;
}


// copy the parts of this CTA's chunk [lo, hi) that peers need into their ghost regions (peer stores)
__device__ __forceinline__ void push_chunk(const PushDesc &pd, int lo, int hi, int tid, int nthreads)
{
    for (int pi = 0; pi < pd.npeers; ++pi) {
        const PushRun *runs = pd.runs[pi];
        const int nr = pd.nruns[pi];
        int a = 0, b = nr;                       // first run that ends after lo
        while (a < b) {
            const int m = (a + b) >> 1;
            if (runs[m].src + runs[m].len <= lo) a = m + 1; else b = m;
        }
        for (int ri = a; ri < nr; ++ri) {
            const PushRun r = runs[ri];
            if (r.src >= hi) break;
            const int s = max(r.src, lo), e = min(r.src + r.len, hi);
            double *d = pd.dst[pi] + ((long long)r.dst_off - (long long)r.src);
            // 8 loads in flight, then 8 peer stores: a one-element loop pays an L2 round trip per element because
            // the stores (possible aliases) pin the loads in program order
            int i = s + tid;
            for (; i + 7 * nthreads < e; i += 8 * nthreads) {
                double t[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) t[u] = __ldcg(pd.src + i + u * nthreads);
#pragma unroll
                for (int u = 0; u < 8; ++u) d[i + u * nthreads] = t[u];
            }
            for (; i < e; i += nthreads) d[i] = __ldcg(pd.src + i);
        }
    }
}


// does the row range [lo, hi) contain anything a peer needs?  (decides which CTAs pay for a system-scope fence)
__device__ __forceinline__ bool push_touches(const PushDesc &pd, int lo, int hi)
{
    for (int pi = 0; pi < pd.npeers; ++pi) {
        const PushRun *runs = pd.runs[pi];
        int a = 0, b = pd.nruns[pi];
        while (a < b) {
            const int m = (a + b) >> 1;
            if (runs[m].src + runs[m].len <= lo) a = m + 1; else b = m;
        }
        if (a < pd.nruns[pi] && runs[a].src < hi) return true;
    }
    return false;
}

} // namespace bicg
