// Block-wide reductions of 64-bit values shared by the nuclear kernels (nuclear.cu, nuclear_tomo.cu).
#pragma once

namespace epid {
namespace nm {

struct OpMax {
    template <class T>
    __device__ T operator()(T a, T b) const { return a > b ? a : b; }
};
struct OpMin {
    template <class T>
    __device__ T operator()(T a, T b) const { return a < b ? a : b; }
};
struct OpSum {
    template <class T>
    __device__ T operator()(T a, T b) const { return a + b; }
};

// block-wide reduction of a 64-bit value; every thread gets the result
template <class T, class Op>
__device__ T block_reduce(T v, Op op, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, (T)__shfl_xor_sync(0xffffffffu, (unsigned long long)v, o));
    __syncthreads();                                        // red[] may still be read by the previous reduction
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = (unsigned long long)v;
    __syncthreads();
    T r = (T)red[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) r = op(r, (T)red[k]);
    return r;
}

}  // namespace nm
}  // namespace epid
