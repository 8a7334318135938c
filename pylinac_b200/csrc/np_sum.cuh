// numpy's pairwise float64 sum (pairwise_sum in numpy's loops) on the host and the device, in numpy's exact tree:
//   n < 8:     sequential from -0.0;
//   n <= 128:  eight strided accumulators r[k] += x[i + k], combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest in sequence;
//   otherwise: pw(x, n2) + pw(x + n2, n - n2) with n2 = n/2 - (n/2) % 8.
// np.sum of a C-contiguous array is 0 + pw(the flattened array); nanmean sums the array with nan set to 0.  The accumulator A is the
// array's own float type (float32 arrays sum in float32); it defaults to double.
//
// pw() is the serial evaluation.  block_pw() is a leaf-parallel one for a CTA of 2^D threads: thread t evaluates the subtree reached
// by the D bits of t (a node that is a leaf above depth D stays on the path of 0 bits; the other paths are empty, +0.0), then the
// slots are added pairwise level by level, which is the tree's own order.  Adding an empty +0.0 slot is exact for sums >= +0.0.
#pragma once

#include <cstdint>

#ifdef __CUDACC__
#define NP_HD __host__ __device__
#else
#define NP_HD
#endif

namespace epid {
namespace np {

constexpr long long PW_BLOCK = 128;

NP_HD inline long long pw_split(long long n) {
    long long n2 = n / 2;
    return n2 - n2 % 8;
}

// one leaf (n <= 128) of elements x(i0) .. x(i0 + n - 1)
template <class X, class A = double>
NP_HD inline A pw_leaf(const X& x, long long i0, long long n) {
    if (n < 8) {
        A res = -0.0;
        for (long long i = 0; i < n; i++) res += x(i0 + i);
        return res;
    }
    A r[8];
    for (int k = 0; k < 8; k++) r[k] = x(i0 + k);
    long long i = 8;
    for (; i < n - n % 8; i += 8)
        for (int k = 0; k < 8; k++) r[k] += x(i0 + i + k);
    A res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += x(i0 + i);
    return res;
}

// pw over x(i0) .. x(i0 + n - 1): the recursion with an explicit stack (its depth is below 64 for any n < 2^63)
template <class X, class A = double>
NP_HD inline A pw(const X& x, long long i0, long long n) {
    long long s[64], m[64];
    A left[64];
    int stage[64];
    int top = 0;
    s[0] = i0;
    m[0] = n;
    stage[0] = 0;
    A ret = 0.0;
    for (;;) {
        if (stage[top] == 0 && m[top] <= PW_BLOCK) {
            ret = pw_leaf<X, A>(x, s[top], m[top]);
        } else if (stage[top] == 0) {
            stage[top] = 1;
            s[top + 1] = s[top];
            m[top + 1] = pw_split(m[top]);
            stage[top + 1] = 0;
            top++;
            continue;
        } else if (stage[top] == 1) {
            const long long n2 = pw_split(m[top]);
            left[top] = ret;
            stage[top] = 2;
            s[top + 1] = s[top] + n2;
            m[top + 1] = m[top] - n2;
            stage[top + 1] = 0;
            top++;
            continue;
        } else {
            ret = left[top] + ret;
        }
        if (top == 0) return ret;
        top--;
    }
}

// the subtree of slot t (D bits, most significant first) of the tree over [0, n): its first element and length; len < 0: empty slot
NP_HD inline void pw_slot(long long n, int t, int D, long long* start, long long* len) {
    long long s = 0, m = n;
    for (int d = D - 1; d >= 0; d--) {
        const int bit = (t >> d) & 1;
        if (m <= PW_BLOCK) {
            if (bit) {
                *start = 0;
                *len = -1;
                return;
            }
            continue;
        }
        const long long n2 = pw_split(m);
        if (bit) {
            s += n2;
            m -= n2;
        } else {
            m = n2;
        }
    }
    *start = s;
    *len = m;
}

#ifdef __CUDACC__
// pw over x(0) .. x(n - 1) by a whole CTA of 2^D = blockDim.x threads; slots: 2^D accumulators of shared memory.  Every thread gets
// the sum.
template <class X, class A>
__device__ A block_pw(const X& x, long long n, int D, A* slots) {
    long long s, m;
    pw_slot(n, threadIdx.x, D, &s, &m);
    A v = m < 0 ? (A)0.0 : pw<X, A>(x, s, m);
    __syncthreads();                              // slots may still be read by a previous call
    slots[threadIdx.x] = v;
    for (int level = D - 1; level >= 0; level--) {
        __syncthreads();
        const int t = threadIdx.x;
        if (t < (1 << level)) v = slots[2 * t] + slots[2 * t + 1];
        __syncthreads();
        if (t < (1 << level)) slots[t] = v;
    }
    __syncthreads();
    return slots[0];
}
#endif

}  // namespace np
}  // namespace epid
