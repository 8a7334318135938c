// The frame stages of get_fov and the FOV uniformities (pylinac.nuclear, nuclear.py:158-271 and 457-481) shared by k_nm_frame
// (nuclear.cu), k_tu_frame (nuclear_tu.cu) and k_nt_slices (nuclear_tomo.cu), and the host code around those kernels.  Every stage
// runs on a whole CTA over one frame of hb x wb pixels held in two int planes P and A (shared memory or a global workspace) and
// decides on `value > 0` only, so it is the same for integer and float64 frames.  Each stage ends with the CTA synchronised.
#pragma once

#include <climits>
#include <cmath>

#include "ccl.cuh"
#include "common.cuh"

namespace epid {
namespace nm {

constexpr int NM_BIG = 1 << 20;        // column distance of a pixel with no background above / below it
// the largest bin: 16 * 65535 * 64^2 < 2^32 keeps k_nm_frame's S a uint32, and each of k_tu_bin's rows stays one pairwise leaf
constexpr int NM_MAX_BIN = 64;

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

// remove_small_objects(min_size=2), connectivity 1: a foreground pixel (value > 0) without a 4-neighbour in the foreground goes.  On
// exit P[p] is p for a kept pixel and -1 otherwise, and val[p] is 0 where P[p] is -1; emit(p, val[p]) sees each pixel's final value.
template <class V, class Emit>
__device__ __forceinline__ void remove_stray_pixels(V* val, int* P, int hb, int wb, Emit emit) {
    const int N = hb * wb, tid = threadIdx.x, nt = blockDim.x;
    for (int p = tid; p < N; p += nt) {
        const int i = p / wb, j = p - i * wb;
        const bool nb = (i > 0 && val[p - wb] > 0) || (i < hb - 1 && val[p + wb] > 0) || (j > 0 && val[p - 1] > 0) ||
                        (j < wb - 1 && val[p + 1] > 0);
        P[p] = val[p] > 0 && nb ? p : -1;
    }
    __syncthreads();
    for (int p = tid; p < N; p += nt) {
        if (P[p] < 0) val[p] = 0;
        emit(p, val[p]);
    }
    __syncthreads();
}

// 4-connected labelling of the foreground (P[p] = p, background -1 on entry): on exit P[p] is the component's root, the smallest index
// of the component (skimage's raster label order), and A[root] its area.
__device__ __forceinline__ void label_areas(int* P, int* A, int hb, int wb) {
    const int N = hb * wb, tid = threadIdx.x, nt = blockDim.x;
    for (int p = tid; p < N; p += nt) {
        if (P[p] < 0) continue;
        const int i = p / wb, j = p - i * wb;
        ccl_join(P, p, j, i, wb, false);
    }
    __syncthreads();
    for (int p = tid; p < N; p += nt) {
        A[p] = 0;
        if (P[p] >= 0) P[p] = gl_find(P, p);
    }
    __syncthreads();
    for (int p = tid; p < N; p += nt)
        if (P[p] >= 0) atomicAdd(&A[P[p]], 1);
    __syncthreads();
}

struct Component {
    int root;                        // the smallest index of the component
    int area;                        // 0: there is no component
    int longest;                     // the longer side of its bounding box
    unsigned long long rsum, csum;   // the exact sums of its pixels' row and column indices
};

// the largest component, on ties the lowest label, i.e. the smallest root (Python's max() keeps the first)
__device__ __forceinline__ Component largest_component(const int* P, const int* A, int hb, int wb, unsigned long long* red) {
    const int N = hb * wb, tid = threadIdx.x, nt = blockDim.x;
    unsigned long long key = 0;
    for (int p = tid; p < N; p += nt) {
        if (P[p] != p) continue;
        const unsigned long long k = ((unsigned long long)A[p] << 32) | (0xffffffffu - (uint32_t)p);
        key = k > key ? k : key;
    }
    key = block_reduce(key, OpMax(), red);
    Component c = {};
    if (key == 0) return c;
    c.root = (int)(0xffffffffu - (uint32_t)key);
    c.area = (int)(key >> 32);
    long long rmin = LLONG_MAX, rmax = -1, cmin = LLONG_MAX, cmax = -1;
    unsigned long long rsum = 0, csum = 0;
    for (int p = tid; p < N; p += nt) {
        if (P[p] != c.root) continue;
        const int i = p / wb, j = p - i * wb;
        rmin = min(rmin, (long long)i);
        rmax = max(rmax, (long long)i);
        cmin = min(cmin, (long long)j);
        cmax = max(cmax, (long long)j);
        rsum += i;
        csum += j;
    }
    rmin = block_reduce(rmin, OpMin(), red);
    rmax = block_reduce(rmax, OpMax(), red);
    cmin = block_reduce(cmin, OpMin(), red);
    cmax = block_reduce(cmax, OpMax(), red);
    c.rsum = block_reduce(rsum, OpSum(), red);
    c.csum = block_reduce(csum, OpSum(), red);
    c.longest = (int)max(rmax - rmin + 1, cmax - cmin + 1);
    return c;
}

// exact squared EDT of the whole binary frame (P >= 0: foreground): column distances into A, then the row-wise minimum of
// dk^2 + g^2 into P (0 on the background).  edt2 (may be null): a copy of the result.
__device__ __forceinline__ void squared_edt(int* P, int* A, int hb, int wb, int32_t* edt2) {
    const int N = hb * wb, tid = threadIdx.x, nt = blockDim.x;
    for (int j = tid; j < wb; j += nt) {
        int g = NM_BIG;
        for (int i = 0; i < hb; i++) {
            const int p = i * wb + j;
            g = P[p] >= 0 ? min(g + 1, NM_BIG) : 0;
            A[p] = g;
        }
        g = NM_BIG;
        for (int i = hb - 1; i >= 0; i--) {
            const int p = i * wb + j;
            g = P[p] >= 0 ? min(g + 1, NM_BIG) : 0;
            A[p] = min(A[p], g);
        }
    }
    __syncthreads();
    for (int p = tid; p < N; p += nt) {      // each thread reads and writes only its own P[p]
        if (P[p] < 0) {
            P[p] = 0;
        } else {
            const int i = p / wb, j = p - i * wb;
            const int* g = A + (size_t)i * wb;
            long long best = (long long)g[j] * g[j];
            for (int k = 1; (long long)k * k < best && (j - k >= 0 || j + k < wb); k++) {
                if (j - k >= 0) best = min(best, (long long)k * k + (long long)g[j - k] * g[j - k]);
                if (j + k < wb) best = min(best, (long long)k * k + (long long)g[j + k] * g[j + k]);
            }
            P[p] = (int)min(best, (long long)INT_MAX);
        }
        if (edt2) edt2[p] = P[p];
    }
    __syncthreads();
}

// the K FOV masks of one frame: distance > erosion / 2  <=>  4 d^2 > erosion^2 (every pixel when the erosion is negative)
template <int K>
struct FovMasks {
    long long e2[K];
    bool all[K];
    __device__ FovMasks(const int* erosion) {
        for (int k = 0; k < K; k++) {
            e2[k] = (long long)erosion[k] * erosion[k];
            all[k] = erosion[k] < 0;
        }
    }
    __device__ bool operator()(const int* edt2, int p, int k) const { return all[k] || 4LL * edt2[p] > e2[k]; }
};

// (max - min) / (max + min) x 100 as the reference evaluates it on the frame's values: exact integers rounded once for the integer
// frame S (the 1/16 of S / 16 cancels exactly), float64 in numpy's order for a float64 frame
__device__ __forceinline__ double michelson100(uint32_t mx, uint32_t mn) {
    return (double)(mx - mn) / (double)((unsigned long long)mx + mn) * 100.0;
}
__device__ __forceinline__ double michelson100(double mx, double mn) { return (mx - mn) / (mx + mn) * 100.0; }
__device__ __forceinline__ uint32_t value_max(uint32_t) { return UINT_MAX; }
__device__ __forceinline__ double value_max(double) { return INFINITY; }
// an order-preserving 64-bit key of a value >= 0
__device__ __forceinline__ unsigned long long value_key(uint32_t v) { return v; }
__device__ __forceinline__ unsigned long long value_key(double v) { return (unsigned long long)__double_as_longlong(v); }

// The uniformities of the K FOVs of a frame of values V (> 0: foreground) and its squared EDT: per FOV the non-zero pixel count,
// integral uniformity with the first raster index of the max / min, and per (FOV, axis) the differential uniformity: windows of `win`
// pixels along axis 0 (a = 0) and axis 1 (a = 1) that hold at least one non-zero FOV pixel, their count, the max of the x100 values and
// its first (i, j) in row-major order.  masks (may be null): the K masks, [K][hb][wb].  R: a result row with n_fov[K], iu[K],
// max_index[K], min_index[K], du_count[2K], du_max[2K], du_index[2K].
template <int K, class V, class R>
__device__ __forceinline__ void fov_uniformity(const V* val, const int* edt2, const FovMasks<K>& in_fov, int hb, int wb, int win,
                                               uint8_t* masks, unsigned long long* red, R& r) {
    const int N = hb * wb, tid = threadIdx.x, nt = blockDim.x;
    unsigned long long mxk[K], mnk[K], nfov[K];
    for (int k = 0; k < K; k++) {
        mxk[k] = 0;
        mnk[k] = ~0ull;
        nfov[k] = 0;
    }
    for (int p = tid; p < N; p += nt) {
        for (int k = 0; k < K; k++) {
            const bool m = in_fov(edt2, p, k);
            if (masks) masks[(size_t)k * N + p] = m;
            if (!m || !(val[p] > 0)) continue;
            if constexpr (sizeof(V) == 4) {                                   // value and index packed in one key
                const unsigned long long hi = value_key(val[p]) << 32;
                mxk[k] = max(mxk[k], hi | (0xffffffffu - (uint32_t)p));      // max value, first index
                mnk[k] = min(mnk[k], hi | (uint32_t)p);                       // min value, first index
            } else {
                mxk[k] = max(mxk[k], value_key(val[p]));
                mnk[k] = min(mnk[k], value_key(val[p]));
            }
            nfov[k]++;
        }
    }
    for (int k = 0; k < K; k++) {
        mxk[k] = block_reduce(mxk[k], OpMax(), red);
        mnk[k] = block_reduce(mnk[k], OpMin(), red);
        nfov[k] = block_reduce(nfov[k], OpSum(), red);
        r.n_fov[k] = (int)nfov[k];
        if (!nfov[k]) continue;
        if constexpr (sizeof(V) == 4) {
            const uint32_t smx = (uint32_t)(mxk[k] >> 32), smn = (uint32_t)(mnk[k] >> 32);
            r.max_index[k] = (int)(0xffffffffu - (uint32_t)mxk[k]);
            r.min_index[k] = (int)(uint32_t)mnk[k];
            r.iu[k] = michelson100(smx, smn);
        } else {                                                              // the first index of each extreme, a second pass
            const double vmx = __longlong_as_double((long long)mxk[k]), vmn = __longlong_as_double((long long)mnk[k]);
            unsigned long long imx = ~0ull, imn = ~0ull;
            for (int p = tid; p < N; p += nt) {
                if (!in_fov(edt2, p, k)) continue;
                if (val[p] == vmx) imx = min(imx, (unsigned long long)p);
                if (val[p] == vmn) imn = min(imn, (unsigned long long)p);
            }
            r.max_index[k] = (int)block_reduce(imx, OpMin(), red);
            r.min_index[k] = (int)block_reduce(imn, OpMin(), red);
            r.iu[k] = michelson100(vmx, vmn);
        }
    }

    for (int k = 0; k < K; k++) {
        for (int a = 0; a < 2; a++) {
            const int ni = a == 0 ? hb - win + 1 : hb, nj = a == 0 ? wb : wb - win + 1;
            const int step = a == 0 ? wb : 1;
            const long long npos = ni > 0 && nj > 0 ? (long long)ni * nj : 0;
            unsigned long long vbest = 0, cnt = 0;
            for (long long q = tid; q < npos; q += nt) {
                const int i = (int)(q / nj), j = (int)(q - (long long)i * nj);
                V mx = 0, mn = value_max(V());
                for (int t = 0, p = i * wb + j; t < win; t++, p += step) {
                    if (!in_fov(edt2, p, k) || !(val[p] > 0)) continue;
                    mx = max(mx, val[p]);
                    mn = min(mn, val[p]);
                }
                if (mx == 0) continue;
                const double v = michelson100(mx, mn);
                vbest = max(vbest, (unsigned long long)__double_as_longlong(v));   // v >= 0: the bits order like the values
                cnt++;
            }
            vbest = block_reduce(vbest, OpMax(), red);
            cnt = block_reduce(cnt, OpSum(), red);
            unsigned long long pos = ~0ull;
            for (long long q = tid; q < npos && cnt; q += nt) {
                const int i = (int)(q / nj), j = (int)(q - (long long)i * nj);
                V mx = 0, mn = value_max(V());
                for (int t = 0, p = i * wb + j; t < win; t++, p += step) {
                    if (!in_fov(edt2, p, k) || !(val[p] > 0)) continue;
                    mx = max(mx, val[p]);
                    mn = min(mn, val[p]);
                }
                if (mx == 0) continue;
                const double v = michelson100(mx, mn);
                if ((unsigned long long)__double_as_longlong(v) == vbest) {
                    pos = (unsigned long long)i * wb + j;
                    break;                                  // q increases, so the thread's first hit is its smallest position
                }
            }
            pos = block_reduce(pos, OpMin(), red);
            r.du_count[2 * k + a] = (int)cnt;
            if (cnt) {
                r.du_max[2 * k + a] = __longlong_as_double((long long)vbest);
                r.du_index[2 * k + a] = (int)pos;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side of the frame kernels

// uint16 frames, read as volumes of nz slices each; `what` names them in the dtype error
inline int check_volumes(const epid_batch* b, int nz, const char* what) {
    EPID_REQUIRE(b, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(b->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "%s must be uint16 (dtype %d)", what, b->dtype);
    EPID_REQUIRE(nz >= 1 && b->n % nz == 0, EPID_ERR_INVALID, "%d slices do not divide the batch's %d frames", nz, b->n);
    return EPID_OK;
}

// the bin size and uniformity window of the FOV uniformities; *hb x *wb: the binned frame, fewer than max_pixels
inline int check_binning(const epid_batch* b, int bin, int window, long long max_pixels, int* hb, int* wb) {
    EPID_REQUIRE(bin >= 1 && bin <= NM_MAX_BIN && (bin & (bin - 1)) == 0, EPID_ERR_UNSUPPORTED,
                 "bin size %d: expected a power of two up to %d", bin, NM_MAX_BIN);
    EPID_REQUIRE(window >= 1, EPID_ERR_INVALID, "window size %d < 1", window);
    *hb = (b->h + bin - 1) / bin;
    *wb = (b->w + bin - 1) / bin;
    EPID_REQUIRE((long long)*hb * *wb < max_pixels, EPID_ERR_UNSUPPORTED, "binned frame %d x %d is too large", *hb, *wb);
    return EPID_OK;
}

struct FrameScratch {
    char* head;       // the caller's leading buffer
    char* rows;       // the result rows
    char* ws;         // the per-frame workspace; nullptr: each CTA holds its frame in `smem` bytes of dynamic shared memory
    char* extra;      // the caller's trailing buffers
    size_t smem;
};

// Lays out ctx->scratch as [head] [rows] [workspace] [extra] for a kernel that runs one CTA per frame of N pixels at bpp bytes per
// pixel.  The frame goes to dynamic shared memory when it fits beside static_smem bytes of static shared memory, else to a workspace
// of bpp x N bytes per frame.  head, rows and the workspace are each rounded up to 256 bytes.
inline int frame_scratch(epid_ctx* ctx, int n, size_t N, size_t bpp, size_t static_smem, size_t head, size_t rows, size_t extra,
                         FrameScratch* s) {
    int optin = 0;
    EPID_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    const bool fits = bpp * N + static_smem <= (size_t)optin;
    const size_t b_head = align256(head), b_rows = align256(rows), b_ws = fits ? 0 : align256(bpp * N * n);
    int rc = ensure_scratch(ctx, b_head + b_rows + b_ws + extra);
    if (rc != EPID_OK) return rc;
    s->head = (char*)ctx->scratch;
    s->rows = s->head + b_head;
    s->ws = fits ? nullptr : s->rows + b_rows;
    s->extra = s->rows + b_rows + b_ws;
    s->smem = fits ? bpp * N : 0;
    return EPID_OK;
}

// the end of an entry point: check the launches, copy the result rows to the host and wait for them
inline int finish(epid_ctx* ctx, void* dst, const void* src, size_t bytes, const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        set_error("%s failed: %s", what, cudaGetErrorString(e));
        return EPID_ERR_CUDA;
    }
    return EPID_OK;
}

}  // namespace nm
}  // namespace epid
