// CT volumes: the two maximum-intensity projections WinstonLutz.from_cbct takes of a slice stack, and the four pseudo-cardinal
// EPID frames it builds from them (winston_lutz.py:1462-1505).
//
// epid_stack_mip: volume [N][H][W] (slice-major, as the slices are read) -> colmax [W][1][N] and rowmax [H][1][N], i.e.
//   np.stack(images, axis=-1).max(axis=0) and .max(axis=1) in the reference's (W, N) / (H, N) layouts, each row one 1-D signal for
//   epid_zoom.  One read of the volume: CTA (band, slice) streams rows [band rows) of one slice; a warp takes whole rows, so the
//   row maximum is a warp reduction, and every lane keeps the column maxima of its fixed 16-byte column chunks in registers (packed
//   16-bit SIMD max).  The warps' column maxima meet in shared memory; with several bands per slice the last CTA of a slice (atomic
//   ticket) folds the per-band partials.  Integer max: exact.
// epid_cbct_views: zoomed projections (float64 [P][1][N']) -> uint16 frames [2k][N'][P]: per projection np.rot90(z, 1) and its
//   np.fliplr, each value rounded the way scipy.ndimage.zoom writes an integer output (half away from zero, clamped to the source
//   dtype), then stored as the 16 bits array_to_dicom writes with PixelRepresentation 0 (an int16 -1000 reads back as 64536).
#include <algorithm>

#include "common.cuh"

namespace epid {

constexpr int MIP_WARPS = 8;
constexpr int MIP_THREADS = MIP_WARPS * 32;
constexpr int MIP_MAX_W = 2048;      // column maxima of 8 warps x W uint16 in shared memory (32 KB)

template <typename T> struct Mip;
template <> struct Mip<int16_t> {
    static constexpr uint32_t low2 = 0x80008000u;     // two packed -32768
    static __device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) { return __vmaxs2(a, b); }
};
template <> struct Mip<uint16_t> {
    static constexpr uint32_t low2 = 0u;
    static __device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) { return __vmaxu2(a, b); }
};

template <typename T>
__device__ __forceinline__ uint4 max4(uint4 a, uint4 b) {
    return make_uint4(Mip<T>::max2(a.x, b.x), Mip<T>::max2(a.y, b.y), Mip<T>::max2(a.z, b.z), Mip<T>::max2(a.w, b.w));
}

template <typename T>
__device__ __forceinline__ int fold2(uint32_t v) {      // max of the two packed halves, as int
    const T lo = (T)(uint16_t)(v & 0xffffu), hi = (T)(uint16_t)(v >> 16);
    return max((int)lo, (int)hi);
}

// CPL > 0: W % 8 == 0, lane owns 16-byte column chunks lane + 32 k (k < CPL), ROWS rows in flight per warp iteration.
// CPL == 0: any W, 2-byte loads, column maxima kept in shared memory (lane owns columns lane + 32 k).
template <typename T, int CPL>
__global__ void __launch_bounds__(MIP_THREADS) k_stack_mip(const T* __restrict__ vol, int N, int H, int W, int bands, int band_rows,
                                                           T* __restrict__ colmax, T* __restrict__ rowmax, T* __restrict__ partial,
                                                           unsigned* __restrict__ tickets) {
    extern __shared__ __align__(16) unsigned char mip_smem[];
    T* scol = (T*)mip_smem;                              // [MIP_WARPS][W]
    const int n = blockIdx.y, band = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r0 = band * band_rows, r1 = min(H, r0 + band_rows);
    const T* __restrict__ slice = vol + (size_t)n * H * W;
    T* __restrict__ my = scol + (size_t)warp * W;
    const T lowT = (T)(uint16_t)(Mip<T>::low2 & 0xffffu);
    if constexpr (CPL > 0) {
        constexpr int ROWS = CPL >= 8 ? 1 : 8 / CPL;
        const int chunks = W >> 3;
        const uint4 low4 = make_uint4(Mip<T>::low2, Mip<T>::low2, Mip<T>::low2, Mip<T>::low2);
        uint4 cm[CPL];
#pragma unroll
        for (int k = 0; k < CPL; k++) cm[k] = low4;
        for (int rb = r0 + warp * ROWS; rb < r1; rb += MIP_WARPS * ROWS) {
            uint4 v[ROWS][CPL];
#pragma unroll
            for (int q = 0; q < ROWS; q++) {
#pragma unroll
                for (int k = 0; k < CPL; k++) {
                    const int c = lane + 32 * k;
                    v[q][k] = (rb + q < r1 && c < chunks) ? ldg_stream16(slice + (size_t)(rb + q) * W + 8 * c) : low4;
                }
            }
#pragma unroll
            for (int q = 0; q < ROWS; q++) {
                uint32_t m = Mip<T>::low2;
#pragma unroll
                for (int k = 0; k < CPL; k++) {
                    cm[k] = max4<T>(cm[k], v[q][k]);
                    m = Mip<T>::max2(m, Mip<T>::max2(Mip<T>::max2(v[q][k].x, v[q][k].y), Mip<T>::max2(v[q][k].z, v[q][k].w)));
                }
                const int rm = warp_max(fold2<T>(m));
                if (lane == 0 && rb + q < r1) rowmax[(size_t)(rb + q) * N + n] = (T)rm;
            }
        }
#pragma unroll
        for (int k = 0; k < CPL; k++) {
            const int c = lane + 32 * k;
            if (c < chunks) *(uint4*)(my + 8 * c) = cm[k];
        }
    } else {
        for (int c = lane; c < W; c += 32) my[c] = lowT;
        for (int r = r0 + warp; r < r1; r += MIP_WARPS) {
            const T* __restrict__ row = slice + (size_t)r * W;
            int m = (int)lowT;
            for (int c = lane; c < W; c += 32) {
                const T v = row[c];
                m = max(m, (int)v);
                if (v > my[c]) my[c] = v;
            }
            m = warp_max(m);
            if (lane == 0) rowmax[(size_t)r * N + n] = (T)m;
        }
    }
    __syncthreads();
    T* dst = bands == 1 ? nullptr : partial + ((size_t)n * bands + band) * W;
    for (int c = threadIdx.x; c < W; c += MIP_THREADS) {
        T m = scol[c];
#pragma unroll
        for (int w = 1; w < MIP_WARPS; w++) m = max(m, scol[(size_t)w * W + c]);
        if (bands == 1) colmax[(size_t)c * N + n] = m;
        else dst[c] = m;
    }
    if (bands == 1) return;
    __shared__ int last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(&tickets[n], 1u) == (unsigned)(bands - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    const T* src = partial + (size_t)n * bands * W;
    for (int c = threadIdx.x; c < W; c += MIP_THREADS) {
        T m = lowT;
        for (int b = 0; b < bands; b++) m = max(m, (T)__ldcg((const short*)(src + (size_t)b * W + c)));
        colmax[(size_t)c * N + n] = m;
    }
}

template <typename T>
static cudaError_t launch_mip(epid_ctx* ctx, const epid_batch* v, int bands, int band_rows, T* colmax, T* rowmax, T* partial,
                              unsigned* tickets) {
    const int N = v->n, H = v->h, W = v->w;
    const dim3 grid(bands, N);
    const size_t smem = sizeof(T) * MIP_WARPS * W;
    const T* src = (const T*)v->dptr;
    const int chunks = W / 8;
    if (W % 8 == 0 && chunks <= 32) k_stack_mip<T, 1><<<grid, MIP_THREADS, smem, ctx->stream>>>(src, N, H, W, bands, band_rows, colmax, rowmax, partial, tickets);
    else if (W % 8 == 0 && chunks <= 64) k_stack_mip<T, 2><<<grid, MIP_THREADS, smem, ctx->stream>>>(src, N, H, W, bands, band_rows, colmax, rowmax, partial, tickets);
    else if (W % 8 == 0 && chunks <= 128) k_stack_mip<T, 4><<<grid, MIP_THREADS, smem, ctx->stream>>>(src, N, H, W, bands, band_rows, colmax, rowmax, partial, tickets);
    else if (W % 8 == 0) k_stack_mip<T, 8><<<grid, MIP_THREADS, smem, ctx->stream>>>(src, N, H, W, bands, band_rows, colmax, rowmax, partial, tickets);
    else k_stack_mip<T, 0><<<grid, MIP_THREADS, smem, ctx->stream>>>(src, N, H, W, bands, band_rows, colmax, rowmax, partial, tickets);
    ctx->launches++;
    return cudaGetLastError();
}

// scipy.ndimage ni_interpolation.c, integer output of an interpolated double: t + 0.5 (t - 0.5 below zero for signed types),
// clamped to the type's range, then the C cast (truncation toward zero)
template <typename T>
__device__ __forceinline__ uint16_t zoom_out_bits(double t);
template <>
__device__ __forceinline__ uint16_t zoom_out_bits<int16_t>(double t) {
    t = t > 0 ? t + 0.5 : t - 0.5;
    t = t > 32767.0 ? 32767.0 : t;
    t = t < -32768.0 ? -32768.0 : t;
    return (uint16_t)(int16_t)(int)t;
}
template <>
__device__ __forceinline__ uint16_t zoom_out_bits<uint16_t>(double t) {
    t = t > 0 ? t + 0.5 : 0.0;
    t = t > 65535.0 ? 65535.0 : t;
    return (uint16_t)(int)t;
}

// frame 2 p = rot90(z_p, 1): out[i][j] = z_p[j][N' - 1 - i]; frame 2 p + 1 = its fliplr: out[i][j] = z_p[P - 1 - j][N' - 1 - i]
template <typename T>
__global__ void k_cbct_views(const double* __restrict__ z0, const double* __restrict__ z1, int P, int Np, uint16_t* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
    if (j >= P || i >= Np) return;
    const double* __restrict__ z = f < 2 ? z0 : z1;
    const int src = (f & 1) ? P - 1 - j : j;
    out[((size_t)f * Np + i) * P + j] = zoom_out_bits<T>(z[(size_t)src * Np + (Np - 1 - i)]);
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_stack_mip(epid_ctx* ctx, const epid_batch* volume, epid_batch** colmax, epid_batch** rowmax) {
    EPID_REQUIRE(ctx && volume && colmax && rowmax, EPID_ERR_INVALID, "NULL argument");
    *colmax = *rowmax = nullptr;
    EPID_REQUIRE(volume->dtype == EPID_I16 || volume->dtype == EPID_U16, EPID_ERR_UNSUPPORTED,
                 "stack projection: dtype %d is not supported (int16 or uint16 slices)", volume->dtype);
    const int N = volume->n, H = volume->h, W = volume->w;
    EPID_REQUIRE(N >= 1 && H >= 1 && W >= 1, EPID_ERR_INVALID, "empty volume");
    EPID_REQUIRE(W <= MIP_MAX_W, EPID_ERR_UNSUPPORTED, "stack projection: slices wider than %d pixels are not supported", MIP_MAX_W);
    EPID_CUDA(cudaSetDevice(ctx->device));
    // bands per slice: enough CTAs to cover every SM several times over, at least 64 rows per band
    int bands = (16 * ctx->sm_count + N - 1) / N;
    bands = std::max(1, std::min(bands, (H + 63) / 64));
    const int band_rows = (H + bands - 1) / bands;
    bands = (H + band_rows - 1) / band_rows;
    const size_t pbytes = bands > 1 ? sizeof(uint16_t) * (size_t)N * bands * W : 0;
    const size_t poff = 256 * ((sizeof(unsigned) * (size_t)N + 255) / 256);
    int rc = EPID_OK;
    if (bands > 1) {
        rc = ensure_scratch(ctx, poff + pbytes);
        if (rc != EPID_OK) return rc;
    }
    unsigned* tickets = bands > 1 ? (unsigned*)ctx->scratch : nullptr;
    void* partial = bands > 1 ? (void*)((char*)ctx->scratch + poff) : nullptr;
    rc = epid_batch_alloc(ctx, volume->dtype, W, 1, N, colmax);
    if (rc == EPID_OK) rc = epid_batch_alloc(ctx, volume->dtype, H, 1, N, rowmax);
    cudaError_t e = cudaSuccess;
    if (rc == EPID_OK) {
        if (bands > 1) e = cudaMemsetAsync(tickets, 0, sizeof(unsigned) * N, ctx->stream);
        if (e == cudaSuccess) {
            if (volume->dtype == EPID_I16)
                e = launch_mip<int16_t>(ctx, volume, bands, band_rows, (int16_t*)(*colmax)->dptr, (int16_t*)(*rowmax)->dptr, (int16_t*)partial, tickets);
            else
                e = launch_mip<uint16_t>(ctx, volume, bands, band_rows, (uint16_t*)(*colmax)->dptr, (uint16_t*)(*rowmax)->dptr, (uint16_t*)partial, tickets);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { set_error("stack projection failed: %s", cudaGetErrorString(e)); rc = EPID_ERR_CUDA; }
    }
    if (rc != EPID_OK) {
        epid_batch_free(*colmax);
        epid_batch_free(*rowmax);
        *colmax = *rowmax = nullptr;
    }
    return rc;
}

extern "C" int32_t epid_cbct_views(epid_ctx* ctx, const epid_batch* z0, const epid_batch* z1, int32_t src_dtype, epid_batch** out) {
    EPID_REQUIRE(ctx && z0 && out, EPID_ERR_INVALID, "NULL argument");
    *out = nullptr;
    EPID_REQUIRE(src_dtype == EPID_I16 || src_dtype == EPID_U16, EPID_ERR_UNSUPPORTED,
                 "CBCT views: source dtype %d is not supported (int16 or uint16)", src_dtype);
    EPID_REQUIRE(z0->dtype == EPID_F64 && z0->h == 1, EPID_ERR_INVALID, "CBCT views take float64 [P][1][N'] projections");
    EPID_REQUIRE(!z1 || (z1->dtype == EPID_F64 && z1->h == 1 && z1->n == z0->n && z1->w == z0->w), EPID_ERR_INVALID,
                 "the two projections of one CBCT view batch must have the same shape");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int P = z0->n, Np = z0->w, frames = z1 ? 4 : 2;
    int rc = epid_batch_alloc(ctx, EPID_U16, frames, Np, P, out);
    if (rc != EPID_OK) return rc;
    const dim3 block(32, 8), grid((P + 31) / 32, (Np + 7) / 8, frames);
    const double* a = (const double*)z0->dptr;
    const double* b = z1 ? (const double*)z1->dptr : nullptr;
    if (src_dtype == EPID_I16) k_cbct_views<int16_t><<<grid, block, 0, ctx->stream>>>(a, b, P, Np, (uint16_t*)(*out)->dptr);
    else k_cbct_views<uint16_t><<<grid, block, 0, ctx->stream>>>(a, b, P, Np, (uint16_t*)(*out)->dptr);
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        set_error("CBCT views failed: %s", cudaGetErrorString(e));
        epid_batch_free(*out);
        *out = nullptr;
        return EPID_ERR_CUDA;
    }
    return EPID_OK;
}
