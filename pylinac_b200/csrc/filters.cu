// Shared-memory tiled stencils.
//
// Median: scipy.ndimage.median_filter(a, size=k) as array_utils.filter calls it (core/array_utils.py:131): full k x k
// footprint, mode='reflect', rank (k*k)/2 of the sorted window (the UPPER median for even k), window offsets
// -(k/2) .. k-1-(k/2) on both axes, dtype preserved.  Every dtype selects the rank the same way: bisection over an
// order-preserving unsigned key (MedKey), counting the window elements <= mid at each step.  A frame of one row (a 1-D
// profile, or a 2-D frame of height 1) runs k_median_row: its k x k window holds k copies of each of k samples, so rank
// k*k/2 is rank k/2 of the k-wide row window.  Tiles are sized per call, (32 + k - 1) x (8 + k - 1) keys for frames and
// 256 + k - 1 keys for rows, up to the device's opt-in shared memory per block; a size no tile can hold is refused.
//
// correlate1d: scipy's symmetric / anti-symmetric summation order in fp64, mode='reflect' (or 'nearest' for the float64 passes
// of ct.cu), per-pass cast to the input dtype.  The weights live in device memory allocated for the call on the context's stream, so any radius runs and two
// contexts on one device never share them.
#include <type_traits>

#include "filters.cuh"

namespace epid {

constexpr int MED_TW = 32, MED_TH = 8;

__device__ __forceinline__ int reflect_idx(int i, int n) {
    // scipy 'reflect': d c b a | a b c d | d c b a
    while (i < 0 || i >= n) {
        if (i < 0) i = -i - 1;
        if (i >= n) i = 2 * n - 1 - i;
    }
    return i;
}

#define EPID_CSWAP(a, b) { const uint32_t _lo = min(a, b); b = max(a, b); a = _lo; }

// Order-preserving unsigned keys: a < b (numpy's order; -0 before +0) <=> key(a) < key(b).  K is the tile element type,
// MAX the largest key the dtype can produce (the bisection's upper bound: 8 steps for uint8, 64 for the 8-byte dtypes).
template <typename T> struct MedKey;
template <> struct MedKey<uint8_t> {
    using K = uint16_t; static constexpr uint64_t MAX = 0xFF;
    static __device__ __forceinline__ K key(uint8_t v) { return v; }
    static __device__ __forceinline__ uint8_t val(uint64_t k) { return (uint8_t)k; }
};
template <> struct MedKey<uint16_t> {
    using K = uint16_t; static constexpr uint64_t MAX = 0xFFFF;
    static __device__ __forceinline__ K key(uint16_t v) { return v; }
    static __device__ __forceinline__ uint16_t val(uint64_t k) { return (uint16_t)k; }
};
template <> struct MedKey<int16_t> {
    using K = uint16_t; static constexpr uint64_t MAX = 0xFFFF;
    static __device__ __forceinline__ K key(int16_t v) { return (uint16_t)v ^ 0x8000u; }
    static __device__ __forceinline__ int16_t val(uint64_t k) { return (int16_t)(uint16_t)(k ^ 0x8000u); }
};
template <> struct MedKey<int32_t> {
    using K = uint32_t; static constexpr uint64_t MAX = 0xFFFFFFFFull;
    static __device__ __forceinline__ K key(int32_t v) { return (uint32_t)v ^ 0x80000000u; }
    static __device__ __forceinline__ int32_t val(uint64_t k) { return (int32_t)((uint32_t)k ^ 0x80000000u); }
};
template <> struct MedKey<long long> {
    using K = uint64_t; static constexpr uint64_t MAX = ~0ull;
    static __device__ __forceinline__ K key(long long v) { return (uint64_t)v ^ 0x8000000000000000ull; }
    static __device__ __forceinline__ long long val(uint64_t k) { return (long long)(k ^ 0x8000000000000000ull); }
};
template <> struct MedKey<float> {
    using K = uint32_t; static constexpr uint64_t MAX = 0xFFFFFFFFull;
    static __device__ __forceinline__ K key(float v) { const uint32_t b = __float_as_uint(v); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
    static __device__ __forceinline__ float val(uint64_t k) { const uint32_t b = (uint32_t)k; return __uint_as_float((b & 0x80000000u) ? (b & 0x7FFFFFFFu) : ~b); }
};
template <> struct MedKey<double> {
    using K = uint64_t; static constexpr uint64_t MAX = ~0ull;
    static __device__ __forceinline__ K key(double v) {
        const uint64_t b = (uint64_t)__double_as_longlong(v);
        return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
    }
    static __device__ __forceinline__ double val(uint64_t k) {
        return __longlong_as_double((long long)((k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
    }
};

// Smallest key v with #{window <= v} >= need, for the kh x kw window whose top-left element is win[0] (row stride tw).
// C is the bisection's arithmetic type: 32 bits while the keys fit, 64 bits otherwise.
template <typename C, typename K>
__device__ __forceinline__ C rank_select(const K* win, int tw, int kh, int kw, int need, C hi) {
    C lo = 0;
    while (lo < hi) {
        const C mid = lo + ((hi - lo) >> 1);
        int c = 0;
        for (int j = 0; j < kh; j++)
            for (int i = 0; i < kw; i++) c += (win[j * tw + i] <= mid) ? 1 : 0;
        if (c >= need) hi = mid; else lo = mid + 1;
    }
    return lo;
}

template <int K>
__global__ void __launch_bounds__(MED_TW * MED_TH)
k_median_u16(const FrameRef* __restrict__ src, const FrameRef* __restrict__ dst, const ValueMap* __restrict__ maps,
             const int* __restrict__ select, int H, int W, int kdyn) {
    const int fi = blockIdx.z;
    if (select && !select[fi]) return;
    const int k = K > 0 ? K : kdyn;
    const int off = k / 2;
    const int tw = MED_TW + k - 1, th = MED_TH + k - 1;
    extern __shared__ uint16_t tile[];
    const FrameRef s = src[fi];
    const int x0 = blockIdx.x * MED_TW, y0 = blockIdx.y * MED_TH;
    const ValueMap vm = maps ? maps[fi] : ValueMap{0, 0, 0};
    for (int i = threadIdx.x; i < tw * th; i += blockDim.x) {
        const int ty = i / tw, tx = i - ty * tw;
        const int yy = reflect_idx(y0 + ty - off, H), xx = reflect_idx(x0 + tx - off, W);
        uint32_t v = __ldg(s.origin + (size_t)yy * s.pitch + xx);
        if (vm.inv) v = vm.mx + vm.mn - v;
        tile[i] = (uint16_t)v;
    }
    __syncthreads();
    const int lx = threadIdx.x % MED_TW, ly = threadIdx.x / MED_TW;
    const int x = x0 + lx, y = y0 + ly;
    if (x >= W || y >= H) return;
    uint32_t result;
    if (K == 3) {
        uint32_t p[9];
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int i = 0; i < 3; i++) p[j * 3 + i] = tile[(ly + j) * tw + lx + i];
        // 19-exchange median-of-9 network
        EPID_CSWAP(p[1], p[2]); EPID_CSWAP(p[4], p[5]); EPID_CSWAP(p[7], p[8]);
        EPID_CSWAP(p[0], p[1]); EPID_CSWAP(p[3], p[4]); EPID_CSWAP(p[6], p[7]);
        EPID_CSWAP(p[1], p[2]); EPID_CSWAP(p[4], p[5]); EPID_CSWAP(p[7], p[8]);
        EPID_CSWAP(p[0], p[3]); EPID_CSWAP(p[5], p[8]); EPID_CSWAP(p[4], p[7]);
        EPID_CSWAP(p[3], p[6]); EPID_CSWAP(p[1], p[4]); EPID_CSWAP(p[2], p[5]);
        EPID_CSWAP(p[4], p[7]); EPID_CSWAP(p[4], p[2]); EPID_CSWAP(p[6], p[4]);
        EPID_CSWAP(p[4], p[2]);
        result = p[4];
    } else {
        result = rank_select<uint32_t>(tile + ly * tw + lx, tw, k, k, (k * k) / 2 + 1, 65535u);
    }
    const FrameRef d = dst[fi];
    const_cast<uint16_t*>(d.origin)[(size_t)y * d.pitch + x] = (uint16_t)result;
}

static constexpr size_t med_tile_bytes(size_t key_bytes, int k) { return key_bytes * (size_t)(MED_TW + k - 1) * (MED_TH + k - 1); }

// The median tile must fit the opt-in shared memory of one block: refuse a size that does not, naming the limit.
static int median_smem(epid_ctx* ctx, size_t smem, int k) {
    int optin = 0;
    EPID_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    EPID_REQUIRE(smem <= (size_t)optin, EPID_ERR_UNSUPPORTED,
                 "median filter size %d needs a %zu-byte shared-memory tile; the device allows %d bytes per block", k, smem, optin);
    return EPID_OK;
}

int launch_median_u16(epid_ctx* ctx, cudaStream_t stream, const FrameRef* d_src, const FrameRef* d_dst, const ValueMap* d_maps,
                      const int* d_select, int n, int H, int W, int k) {
    EPID_REQUIRE(k >= 1, EPID_ERR_INVALID, "median filter size %d must be >= 1", k);
    dim3 grid((W + MED_TW - 1) / MED_TW, (H + MED_TH - 1) / MED_TH, n);
    const size_t smem = med_tile_bytes(sizeof(uint16_t), k);
    if (k == 3) {
        k_median_u16<3><<<grid, MED_TW * MED_TH, smem, stream>>>(d_src, d_dst, d_maps, d_select, H, W, k);
    } else {
        int rc = median_smem(ctx, smem, k);
        if (rc != EPID_OK) return rc;
        EPID_SMEM_OPT_IN(ctx, k_median_u16<0>, smem);
        k_median_u16<0><<<grid, MED_TW * MED_TH, smem, stream>>>(d_src, d_dst, d_maps, d_select, H, W, k);
    }
    ctx->launches += 1;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

// k x k median of compact frames (every dtype but uint16, which runs k_median_u16)
template <typename T>
__global__ void __launch_bounds__(MED_TW * MED_TH)
k_median_key(const T* __restrict__ in, T* __restrict__ out, int H, int W, int k) {
    using M = MedKey<T>;
    using K = typename M::K;
    using C = typename std::conditional<sizeof(K) <= 4, uint32_t, uint64_t>::type;
    extern __shared__ __align__(8) unsigned char med_raw[];
    K* tile = reinterpret_cast<K*>(med_raw);
    const int fi = blockIdx.z;
    const T* f = in + (size_t)fi * H * W;
    const int off = k / 2;
    const int tw = MED_TW + k - 1, th = MED_TH + k - 1;
    const int x0 = blockIdx.x * MED_TW, y0 = blockIdx.y * MED_TH;
    for (int i = threadIdx.x; i < tw * th; i += blockDim.x) {
        const int ty = i / tw, tx = i - ty * tw;
        tile[i] = M::key(f[(size_t)reflect_idx(y0 + ty - off, H) * W + reflect_idx(x0 + tx - off, W)]);
    }
    __syncthreads();
    const int lx = threadIdx.x % MED_TW, ly = threadIdx.x / MED_TW;
    const int x = x0 + lx, y = y0 + ly;
    if (x >= W || y >= H) return;
    out[(size_t)fi * H * W + (size_t)y * W + x] = M::val(rank_select<C>(tile + ly * tw + lx, tw, k, k, (k * k) / 2 + 1, (C)M::MAX));
}

// median of frames of one row: rank k/2 of the k-wide window (every dtype)
constexpr int MED_ROW = 256;
template <typename T>
__global__ void __launch_bounds__(MED_ROW)
k_median_row(const T* __restrict__ in, T* __restrict__ out, int W, int k) {
    using M = MedKey<T>;
    using K = typename M::K;
    using C = typename std::conditional<sizeof(K) <= 4, uint32_t, uint64_t>::type;
    extern __shared__ __align__(8) unsigned char med_raw[];
    K* tile = reinterpret_cast<K*>(med_raw);
    const T* f = in + (size_t)blockIdx.z * W;
    const int x0 = blockIdx.x * MED_ROW;
    for (int i = threadIdx.x; i < MED_ROW + k - 1; i += MED_ROW) tile[i] = M::key(f[reflect_idx(x0 + i - k / 2, W)]);
    __syncthreads();
    const int x = x0 + threadIdx.x;
    if (x >= W) return;
    out[(size_t)blockIdx.z * W + x] = M::val(rank_select<C>(tile + threadIdx.x, 0, 1, k, k / 2 + 1, (C)M::MAX));
}

template <typename T>
static int run_median(epid_ctx* ctx, const epid_batch* in, epid_batch* out, int k) {
    using K = typename MedKey<T>::K;
    int rc;
    if (in->h == 1) {
        const size_t smem = sizeof(K) * ((size_t)MED_ROW + k - 1);
        if ((rc = median_smem(ctx, smem, k)) != EPID_OK) return rc;
        EPID_SMEM_OPT_IN(ctx, k_median_row<T>, smem);
        k_median_row<T><<<dim3((in->w + MED_ROW - 1) / MED_ROW, 1, in->n), MED_ROW, smem, ctx->stream>>>((const T*)in->dptr, (T*)out->dptr, in->w, k);
    } else if constexpr (std::is_same<T, uint16_t>::value) {
        const int n = in->n;
        if ((rc = ensure_scratch(ctx, 2 * sizeof(FrameRef) * n + 512)) != EPID_OK) return rc;
        FrameRef* src = (FrameRef*)ctx->scratch;
        FrameRef* dst = (FrameRef*)((char*)ctx->scratch + align256(sizeof(FrameRef) * n));
        launch_refs_from_batch(ctx, ctx->stream, (const uint16_t*)in->dptr, n, in->h, in->w, 0, 0, src);
        launch_refs_from_batch(ctx, ctx->stream, (const uint16_t*)out->dptr, n, in->h, in->w, 0, 0, dst);
        return launch_median_u16(ctx, ctx->stream, src, dst, nullptr, nullptr, n, in->h, in->w, k);
    } else {
        const size_t smem = med_tile_bytes(sizeof(K), k);
        if ((rc = median_smem(ctx, smem, k)) != EPID_OK) return rc;
        EPID_SMEM_OPT_IN(ctx, k_median_key<T>, smem);
        dim3 grid((in->w + MED_TW - 1) / MED_TW, (in->h + MED_TH - 1) / MED_TH, in->n);
        k_median_key<T><<<grid, MED_TW * MED_TH, smem, ctx->stream>>>((const T*)in->dptr, (T*)out->dptr, in->h, in->w, k);
    }
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace epid

// ================================================================================================ generic dtypes
namespace epid {

// One 1-D correlation pass along `axis` with scipy.ndimage.correlate1d's symmetric / anti-symmetric summation
// order (ni_filters.c NI_Correlate1D), mode 'reflect' (nearest == 0) or 'nearest' (nearest == 1: a b | a b c d | c d), fp64
// accumulation, result cast to T.
//   sym > 0:  tmp = x[l]*w[r];  for ll = -r..-1: tmp += (x[l+ll] + x[l-ll]) * w[ll+r]
//   sym < 0:  tmp = x[l]*w[r];  for ll = -r..-1: tmp += (x[l+ll] - x[l-ll]) * w[ll+r]
//   sym == 0: tmp = sum_{ll=-r..r} x[l+ll] * w[ll+r]
template <typename T>
__device__ __forceinline__ T cast_from_double(double v) { return (T)v; }
template <> __device__ __forceinline__ uint8_t cast_from_double<uint8_t>(double v) { return (uint8_t)(long long)v; }
template <> __device__ __forceinline__ uint16_t cast_from_double<uint16_t>(double v) { return (uint16_t)(long long)v; }
template <> __device__ __forceinline__ int16_t cast_from_double<int16_t>(double v) { return (int16_t)(long long)v; }
// scipy's (npy_int)double is x86's cvttsd2si: a result outside int32 (or NaN) becomes INT32_MIN; narrower types wrap
template <> __device__ __forceinline__ int32_t cast_from_double<int32_t>(double v) {
    return (v >= -2147483648.0 && v < 2147483648.0) ? (int32_t)v : INT32_MIN;
}

template <typename T>
__global__ void __launch_bounds__(256)
k_correlate1d(const T* __restrict__ in, T* __restrict__ out, const double* __restrict__ c_weights, int H, int W, int axis, int r, int sym,
              int nearest) {
    const int fi = blockIdx.z;
    const T* f = in + (size_t)fi * H * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W) return;
    const int n = axis == 0 ? H : W;
    const int l = axis == 0 ? y : x;
    auto at = [&](int idx) -> double {
        const int j = nearest ? min(max(idx, 0), n - 1) : reflect_idx(idx, n);
        return (double)(axis == 0 ? f[(size_t)j * W + x] : f[(size_t)y * W + j]);
    };
    double tmp;
    if (sym > 0) {
        tmp = at(l) * c_weights[r];
        for (int ll = -r; ll < 0; ll++) tmp += (at(l + ll) + at(l - ll)) * c_weights[ll + r];
    } else if (sym < 0) {
        tmp = at(l) * c_weights[r];
        for (int ll = -r; ll < 0; ll++) tmp += (at(l + ll) - at(l - ll)) * c_weights[ll + r];
    } else {
        tmp = at(l - r) * c_weights[0];
        for (int ll = -r + 1; ll <= r; ll++) tmp += at(l + ll) * c_weights[ll + r];
    }
    out[(size_t)fi * H * W + (size_t)y * W + x] = cast_from_double<T>(tmp);
}

template <typename T>
static int run_correlate(epid_ctx* ctx, const void* in, void* out, int n, int H, int W, int axis, const double* w, int r, int nearest = 0) {
    // symmetry test as in scipy (ni_filters.c): |w[i] - w[2r-i]| <= DBL_EPSILON for all i -> symmetric
    int sym = 0;
    if (r > 0) {
        sym = 1;
        for (int i = 1; i <= r; i++) if (fabs(w[r + i] - w[r - i]) > 2.220446049250313e-16) { sym = 0; break; }
        if (sym == 0) {
            sym = -1;
            for (int i = 1; i <= r; i++) if (fabs(w[r + i] + w[r - i]) > 2.220446049250313e-16) { sym = 0; break; }
        }
    }
    // weights for this pass only, in stream order: a later pass or another context cannot overwrite them before the kernel reads them
    double* d_w = nullptr;
    EPID_CUDA(cudaMallocAsync((void**)&d_w, sizeof(double) * (2 * r + 1), ctx->stream));
    cudaError_t e = cudaMemcpyAsync(d_w, w, sizeof(double) * (2 * r + 1), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        dim3 grid((W + 255) / 256, H, n);
        k_correlate1d<T><<<grid, 256, 0, ctx->stream>>>((const T*)in, (T*)out, d_w, H, W, axis, r, sym, nearest);
        ctx->launches++;
        e = cudaGetLastError();
    }
    const cudaError_t ef = cudaFreeAsync(d_w, ctx->stream);
    EPID_CUDA(e);
    EPID_CUDA(ef);
    return EPID_OK;
}

int correlate1d_f64(epid_ctx* ctx, const double* in, double* out, int n, int H, int W, int axis, const double* w, int r, int nearest) {
    return run_correlate<double>(ctx, in, out, n, H, W, axis, w, r, nearest);
}

static int sync_and_check(epid_ctx* ctx, int rc, epid_batch** out) {
    if (rc == EPID_OK) {
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { set_error("kernel failed: %s", cudaGetErrorString(e)); rc = EPID_ERR_CUDA; }
    }
    if (rc != EPID_OK && out && *out) { epid_batch_free(*out); *out = nullptr; }
    return rc;
}

#define EPID_FDISPATCH(dt, FN, ...)                                                 \
    switch (dt) {                                                                   \
        case EPID_U8: rc = FN<uint8_t>(__VA_ARGS__); break;                         \
        case EPID_U16: rc = FN<uint16_t>(__VA_ARGS__); break;                       \
        case EPID_I16: rc = FN<int16_t>(__VA_ARGS__); break;                        \
        case EPID_I32: rc = FN<int32_t>(__VA_ARGS__); break;                        \
        case EPID_I64: rc = FN<long long>(__VA_ARGS__); break;                      \
        case EPID_F32: rc = FN<float>(__VA_ARGS__); break;                          \
        case EPID_F64: rc = FN<double>(__VA_ARGS__); break;                         \
        default: set_error("unknown dtype %d", dt); rc = EPID_ERR_INVALID;          \
    }

int gaussian_weights(double sigma, std::vector<double>& w, int* radius) {
    // scipy.ndimage._filters._gaussian_kernel1d (order 0), truncate = 4.0
    const int r = (int)(4.0 * sigma + 0.5);
    w.resize(2 * r + 1);
    const double s2 = sigma * sigma;
    double sum = 0.0;
    for (int i = -r; i <= r; i++) { w[i + r] = exp(-0.5 / s2 * (double)(i * i)); }
    for (int i = 0; i < 2 * r + 1; i++) sum += w[i];
    for (int i = 0; i < 2 * r + 1; i++) w[i] /= sum;
    *radius = r;
    return EPID_OK;
}

}  // namespace epid

using namespace epid;

extern "C" {

int32_t epid_median_filter(epid_ctx* ctx, const epid_batch* in, int32_t size, epid_batch** out) {
    EPID_REQUIRE(ctx && in && out, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(size >= 1, EPID_ERR_INVALID, "median filter size must be >= 1");
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = epid_batch_alloc(ctx, in->dtype, in->n, in->h, in->w, out);
    if (rc != EPID_OK) return rc;
    EPID_FDISPATCH(in->dtype, run_median, ctx, in, *out, size);
    return sync_and_check(ctx, rc, out);
}

/* explicit-weights variant used by the python binding so that the weights are the very doubles scipy computes */
int32_t epid_correlate1d_passes(epid_ctx* ctx, const epid_batch* in, const double* weights, int32_t radius, int32_t axes, epid_batch** out) {
    EPID_REQUIRE(ctx && in && out && weights && radius >= 0 && axes >= 1 && axes <= 3, EPID_ERR_INVALID, "bad argument");
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = epid_batch_alloc(ctx, in->dtype, in->n, in->h, in->w, out);
    if (rc != EPID_OK) return rc;
    epid_batch* tmp = nullptr;
    rc = epid_batch_alloc(ctx, in->dtype, in->n, in->h, in->w, &tmp);
    if (rc != EPID_OK) { epid_batch_free(*out); *out = nullptr; return rc; }
    if (axes == 3) {
        EPID_FDISPATCH(in->dtype, run_correlate, ctx, in->dptr, tmp->dptr, in->n, in->h, in->w, 0, weights, radius);
        if (rc == EPID_OK) { EPID_FDISPATCH(in->dtype, run_correlate, ctx, tmp->dptr, (*out)->dptr, in->n, in->h, in->w, 1, weights, radius); }
    } else {
        EPID_FDISPATCH(in->dtype, run_correlate, ctx, in->dptr, (*out)->dptr, in->n, in->h, in->w, axes == 1 ? 0 : 1, weights, radius);
    }
    rc = sync_and_check(ctx, rc, out);
    epid_batch_free(tmp);
    return rc;
}

int32_t epid_gaussian_filter(epid_ctx* ctx, const epid_batch* in, double sigma, epid_batch** out) {
    EPID_REQUIRE(sigma > 0, EPID_ERR_INVALID, "sigma must be positive");
    std::vector<double> w;
    int r = 0;
    gaussian_weights(sigma, w, &r);
    return epid_correlate1d_passes(ctx, in, w.data(), r, 3, out);
}

int32_t epid_sobel(epid_ctx* ctx, const epid_batch* in, int32_t axis, epid_batch** out) {
    EPID_REQUIRE(ctx && in && out, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(axis == 0 || axis == 1 || axis == -1, EPID_ERR_INVALID, "axis must be 0 or 1");
    if (axis == -1) axis = 1;
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = epid_batch_alloc(ctx, in->dtype, in->n, in->h, in->w, out);
    if (rc != EPID_OK) return rc;
    epid_batch* tmp = nullptr;
    rc = epid_batch_alloc(ctx, in->dtype, in->n, in->h, in->w, &tmp);
    if (rc != EPID_OK) { epid_batch_free(*out); *out = nullptr; return rc; }
    // scipy.ndimage.sobel: correlate1d(input, [-1, 0, 1], axis) then correlate1d(., [1, 2, 1], other axis)
    const double d[3] = {-1.0, 0.0, 1.0}, s[3] = {1.0, 2.0, 1.0};
    EPID_FDISPATCH(in->dtype, run_correlate, ctx, in->dptr, tmp->dptr, in->n, in->h, in->w, axis, d, 1);
    if (rc == EPID_OK) { EPID_FDISPATCH(in->dtype, run_correlate, ctx, tmp->dptr, (*out)->dptr, in->n, in->h, in->w, 1 - axis, s, 1); }
    rc = sync_and_check(ctx, rc, out);
    epid_batch_free(tmp);
    return rc;
}

}  // extern "C"
