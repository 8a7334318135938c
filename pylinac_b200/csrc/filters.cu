// Shared-memory tiled stencils.  Median: scipy.ndimage.median_filter(a, size=k) as array_utils.filter calls it
// (core/array_utils.py:131): full k x k footprint, mode='reflect', rank (k*k)/2 of the sorted window (the UPPER
// median for even k), window offsets -(k/2) .. k-1-(k/2) on both axes, dtype preserved.
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
        // rank select by bisection on the 16 value bits: smallest v with #{window <= v} >= rank + 1
        const int need = (k * k) / 2 + 1;
        uint32_t lo = 0, hi = 65535;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            int c = 0;
            for (int j = 0; j < k; j++)
                for (int i = 0; i < k; i++) c += (tile[(ly + j) * tw + lx + i] <= mid) ? 1 : 0;
            if (c >= need) hi = mid; else lo = mid + 1;
        }
        result = lo;
    }
    const FrameRef d = dst[fi];
    const_cast<uint16_t*>(d.origin)[(size_t)y * d.pitch + x] = (uint16_t)result;
}

int launch_median_u16(epid_ctx* ctx, cudaStream_t stream, const FrameRef* d_src, const FrameRef* d_dst, const ValueMap* d_maps,
                      const int* d_select, int n, int H, int W, int k) {
    EPID_REQUIRE(k >= 1 && k <= 31, EPID_ERR_UNSUPPORTED, "median filter size %d outside 1..31", k);
    dim3 grid((W + MED_TW - 1) / MED_TW, (H + MED_TH - 1) / MED_TH, n);
    const size_t smem = sizeof(uint16_t) * (size_t)(MED_TW + k - 1) * (MED_TH + k - 1);
    if (k == 3)
        k_median_u16<3><<<grid, MED_TW * MED_TH, smem, stream>>>(d_src, d_dst, d_maps, d_select, H, W, k);
    else
        k_median_u16<0><<<grid, MED_TW * MED_TH, smem, stream>>>(d_src, d_dst, d_maps, d_select, H, W, k);
    ctx->launches += 1;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace epid

// ================================================================================================ generic dtypes
namespace epid {

// rank-by-counting median for any ordered dtype (used for everything that is not uint16): O(k^4) per pixel,
// exact scipy semantics (element of rank k*k/2 in the sorted window).
template <typename T>
__global__ void __launch_bounds__(MED_TW * MED_TH)
k_median_generic(const T* __restrict__ in, T* __restrict__ out, int H, int W, int k) {
    extern __shared__ unsigned char traw[];
    T* tile = reinterpret_cast<T*>(traw);
    const int fi = blockIdx.z;
    const T* f = in + (size_t)fi * H * W;
    const int off = k / 2;
    const int tw = MED_TW + k - 1, th = MED_TH + k - 1;
    const int x0 = blockIdx.x * MED_TW, y0 = blockIdx.y * MED_TH;
    for (int i = threadIdx.x; i < tw * th; i += blockDim.x) {
        const int ty = i / tw, tx = i - ty * tw;
        tile[i] = f[(size_t)reflect_idx(y0 + ty - off, H) * W + reflect_idx(x0 + tx - off, W)];
    }
    __syncthreads();
    const int lx = threadIdx.x % MED_TW, ly = threadIdx.x / MED_TW;
    const int x = x0 + lx, y = y0 + ly;
    if (x >= W || y >= H) return;
    const int want = (k * k) / 2;
    T result = tile[ly * tw + lx];
    for (int a = 0; a < k * k; a++) {
        const T v = tile[(ly + a / k) * tw + lx + a % k];
        int rank = 0;
        for (int b = 0; b < k * k; b++) {
            const T o = tile[(ly + b / k) * tw + lx + b % k];
            rank += (o < v || (o == v && b < a)) ? 1 : 0;
        }
        if (rank == want) { result = v; break; }
    }
    out[(size_t)fi * H * W + (size_t)y * W + x] = result;
}

// One 1-D correlation pass along `axis` with scipy.ndimage.correlate1d's symmetric / anti-symmetric summation
// order (ni_filters.c NI_Correlate1D), mode='reflect', fp64 accumulation, result cast to T.
//   sym > 0:  tmp = x[l]*w[r];  for ll = -r..-1: tmp += (x[l+ll] + x[l-ll]) * w[ll+r]
//   sym < 0:  tmp = x[l]*w[r];  for ll = -r..-1: tmp += (x[l+ll] - x[l-ll]) * w[ll+r]
//   sym == 0: tmp = sum_{ll=-r..r} x[l+ll] * w[ll+r]
template <typename T>
__device__ __forceinline__ T cast_from_double(double v) { return (T)v; }
template <> __device__ __forceinline__ uint8_t cast_from_double<uint8_t>(double v) { return (uint8_t)(long long)v; }
template <> __device__ __forceinline__ uint16_t cast_from_double<uint16_t>(double v) { return (uint16_t)(long long)v; }
template <> __device__ __forceinline__ int16_t cast_from_double<int16_t>(double v) { return (int16_t)(long long)v; }
template <> __device__ __forceinline__ int32_t cast_from_double<int32_t>(double v) { return (int32_t)(long long)v; }

constexpr int CORR_MAX_TAPS = 513;
__constant__ double c_weights[CORR_MAX_TAPS];

template <typename T>
__global__ void __launch_bounds__(256)
k_correlate1d(const T* __restrict__ in, T* __restrict__ out, int H, int W, int axis, int r, int sym) {
    const int fi = blockIdx.z;
    const T* f = in + (size_t)fi * H * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W) return;
    const int n = axis == 0 ? H : W;
    const int l = axis == 0 ? y : x;
    auto at = [&](int idx) -> double {
        const int j = reflect_idx(idx, n);
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
static int run_correlate(epid_ctx* ctx, const void* in, void* out, int n, int H, int W, int axis, const double* w, int r) {
    EPID_REQUIRE(2 * r + 1 <= CORR_MAX_TAPS, EPID_ERR_UNSUPPORTED, "kernel radius %d too large", r);
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
    EPID_CUDA(cudaMemcpyToSymbolAsync(c_weights, w, sizeof(double) * (2 * r + 1), 0, cudaMemcpyHostToDevice, ctx->stream));
    dim3 grid((W + 255) / 256, H, n);
    k_correlate1d<T><<<grid, 256, 0, ctx->stream>>>((const T*)in, (T*)out, H, W, axis, r, sym);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

template <typename T>
static int run_median_generic(epid_ctx* ctx, const epid_batch* in, epid_batch* out, int k) {
    dim3 grid((in->w + MED_TW - 1) / MED_TW, (in->h + MED_TH - 1) / MED_TH, in->n);
    const size_t smem = sizeof(T) * (size_t)(MED_TW + k - 1) * (MED_TH + k - 1);
    EPID_REQUIRE(smem <= 48 * 1024, EPID_ERR_UNSUPPORTED, "median filter size %d too large for this dtype", k);
    k_median_generic<T><<<grid, MED_TW * MED_TH, smem, ctx->stream>>>((const T*)in->dptr, (T*)out->dptr, in->h, in->w, k);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
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
    if (in->dtype == EPID_U16) {
        const int n = in->n;
        rc = ensure_scratch(ctx, 2 * sizeof(FrameRef) * n + 512);
        if (rc == EPID_OK) {
            FrameRef* src = (FrameRef*)ctx->scratch;
            FrameRef* dst = (FrameRef*)((char*)ctx->scratch + (sizeof(FrameRef) * n + 255) / 256 * 256);
            launch_refs_from_batch(ctx, ctx->stream, (const uint16_t*)in->dptr, n, in->h, in->w, 0, 0, src);
            launch_refs_from_batch(ctx, ctx->stream, (const uint16_t*)(*out)->dptr, n, in->h, in->w, 0, 0, dst);
            rc = launch_median_u16(ctx, ctx->stream, src, dst, nullptr, nullptr, n, in->h, in->w, size);
        }
    } else {
        EPID_FDISPATCH(in->dtype, run_median_generic, ctx, in, *out, size);
    }
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
