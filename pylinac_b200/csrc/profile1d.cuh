// Block-wide 1-D helpers shared by the profile stages of vmat.cu and lightrad.cu (internal interface).
#pragma once
#include "common.cuh"
#include "peaks.cuh"

namespace epid {

#define VM_INF (__longlong_as_double(0x7ff0000000000000LL))

struct OpMin { __device__ static double f(double a, double b) { return fmin(a, b); } };
struct OpMax { __device__ static double f(double a, double b) { return fmax(a, b); } };
struct OpSum { __device__ static double f(double a, double b) { return a + b; } };

template <class Op>
__device__ double blk_reduce(double v, double* red) {      // red: >= 33 doubles of shared memory; result broadcast to every thread
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = Op::f(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = red[0];
        for (int k = 1; k < nw; k++) t = Op::f(t, red[k]);
        red[32] = t;
    }
    __syncthreads();
    return red[32];
}

// FWXMProfile.field_edge_idx: find_peaks(values, fwxm_height, max_number=1) -> left / right interpolated positions
__device__ inline int vm_edges(const double* v, int n, PeakWork& pw, double* l, double* r, double fwxm_height = 0.5) {
    PeakArgs a;
    a.hmin = -VM_INF;
    a.distance = 1;
    a.pmin = -1.0;
    a.wmin = 0.0;
    a.rel_height = 1.0 - fwxm_height;
    a.max_number = 1;
    a.sort_by_height = 0;
    const int c = block_find_peaks(v, n, a, pw);
    __syncthreads();
    if (c < 1) return 2;
    *l = pw.lip[0];
    *r = pw.rip[0];
    return 0;
}

__device__ inline double vm_lerp_at(const double* v, int n, double x) {      // UnivariateSpline(k=1, s=0) through (i, v[i])
    int i = (int)floor(x);
    i = max(0, min(i, n - 2));
    const double u = x - (double)i;
    return v[i] * (1.0 - u) + v[i + 1] * u;
}

}  // namespace epid
