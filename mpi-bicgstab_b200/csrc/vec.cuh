// vec.cuh -- argument block + launch interface of the fused vector-update kernels (vec.cu)
#pragma once
#include "dev.cuh"

namespace bicg {

// a run of consecutive local elements that one peer needs in its ghost region
struct PushRun { int src; int len; int dst_off; };

struct PushDesc {
    int npeers;                              // 0: nothing to push
    const double  *src;                      // the vector being pushed (own part)
    double        *dst[MAX_RANKS - 1];       // peer-mapped base of that vector's ghost region on peer i
    const PushRun *runs[MAX_RANKS - 1];      // runs for peer i, sorted by src, disjoint
    int            nruns[MAX_RANKS - 1];
};

// arena vectors
enum VecId { V_X = 0, V_R, V_RH, V_P, V_S, V_Y, V_W, V_V, V_T, V_B, V_AX, V_COUNT };
// V_Y doubles as z (the CA / pipelined variants call the same storage z)
constexpr int V_Z = V_Y;

// vector roles (pointers to the own part of each arena vector; unused ones are null)
struct VecPtrs {
    double *x, *r, *rh, *p, *s, *y, *z, *w, *v, *t, *b, *ax;
};

struct VecArgs {
    KernelCommon kc;
    VecPtrs v;
    int n;          // local length
    int chunk;      // elements per CTA (multiple of 4)
    PushDesc push;
};

// phases: one fused kernel each.  The reference lines each one replaces are listed in vec.cu.
enum Phase : int {
    PH_BICG_INIT = 0,   // r=b-Ax, r#=r, p=r, (r,r)                 [push p]
    PH_BICG_Q,          // q=r-alpha s                               [push r]
    PH_BICG_XR,         // x+=alpha p+omega q, r=q-omega y, (r,r),(r#,r)
    PH_BICG_P,          // p=r+beta(p-omega s)                       [push p]
    PH_INIT_R,          // r=b-Ax, r#=r, (r,r)                       [push r]
    PH_CA_PS,           // p,s recurrences                           [push s]
    PH_QY,              // q=r-alpha s, y=w-alpha z, (q,y),(y,y)     [push z when asked]
    PH_CA_XR,           // x, r updates, (r,r)                       [push r]
    PH_PIPE_1,          // p,s,z recurrences, q, y, (q,y),(y,y)      [push z]
    PH_PIPE_3,          // x, r, w=y-omega(t-alpha v), 5 dots        [push w]
    PH_RR_P,            // p recurrence only                         [push p]
    PH_RR_X,            // x update only                             [push x]
    PH_RR_R,            // r=b-Ax                                    [push r]
    PH_RR_DOTS,         // 5 dots                                    [push w]
    PH_PUSH,            // push only
    PH_COUNT
};

int launch_vec(int phase, int grid, const VecArgs &a, cudaStream_t st);

} // namespace bicg
