// CT phantom localization (pylinac.ct, ct.py:381-433 Slice.phantom_roi with ct.py:3315-3348 get_regions on its ndarray branch:
// fill_holes=True, threshold="otsu", clip_in_localization=True), for every listed slice of a device-resident int16 / uint16 series.
//
// Per slice, each stage equal bit for bit to the numpy / scipy / skimage call it restates:
//   k_ct_scharr   HU = raw * slope + intercept (float64, two roundings), skimage.filters.scharr of HU (its maximum: the edge check)
//                 and of np.clip(HU, -1000, 1000), each ndimage.convolve pass in NI_Correlate's footprint order, mode 'reflect'
//   correlate1d   skimage.filters.gaussian(sigma=1) = ndimage.gaussian_filter(mode='nearest', truncate=4): filters.cu's passes
//   k_ct_otsu     threshold_otsu: np.histogram's 256 linspace bins and float bin assignment, then the between-class variance argmax
//   k_ct_*        bw = edges > thres; clear_border (8-connected objects reaching the outer buffer_size + 1 rows / columns);
//                 binary_fill_holes (background 4-connected to the outside stays); measure.label (8-connected); per region the
//                 area and exact row / column sums
//   k_ct_select   the region with the smallest |area - catphan_size| (first label on ties) and the 1.3x size check
// Labels are union-find roots within each slice (ccl.cuh): the smallest index of a component, which is skimage's raster label order.
// After the global fill every region's filled_area equals its area (no background is enclosed), so area stands for both.
#include <cfloat>

#include "ccl.cuh"
#include "common.cuh"
#include "filters.cuh"

namespace epid {
namespace {

constexpr int CT_THREADS = 256;
constexpr int CT_SEL_THREADS = 1024;
constexpr int CT_BINS = 256;
// slices per chunk: at most this many pixels, so one chunk's planes stay under 1 GB and its indices in int32
constexpr long long CT_CHUNK_PIXELS = 1ll << 24;
constexpr int CT_MAX_GRID = 65535;      // the largest grid.y / grid.z

__device__ __forceinline__ int reflect1(int i, int n) {      // scipy 'reflect' for an offset of one pixel
    return i < 0 ? -i - 1 : (i >= n ? 2 * n - 1 - i : i);
}

struct SliceIn {
    const void* raw;       // the slice's first pixel
    double slope, intercept;
};

template <typename T>
__device__ __forceinline__ double hu_at(const T* f, int W, int y, int x, double slope, double intercept) {
    return (double)f[(size_t)y * W + x] * slope + intercept;
}

// skimage.filters.scharr of a 3 x 3 neighbourhood v (row-major): per axis ndimage.convolve with the reversed kernel, i.e. correlate
// with its non-zero weights summed from 0.0 in footprint order, then sqrt(a0 * a0 + a1 * a1) / sqrt(2).
__device__ __forceinline__ double scharr3(const double v[9]) {
    const double s = 0.1875, c = 0.625;   // [3, 10, 3] / 16
    double a0 = 0.0;
    a0 += v[0] * -s; a0 += v[1] * -c; a0 += v[2] * -s;
    a0 += v[6] * s;  a0 += v[7] * c;  a0 += v[8] * s;
    double a1 = 0.0;
    a1 += v[0] * -s; a1 += v[2] * s;
    a1 += v[3] * -c; a1 += v[5] * c;
    a1 += v[6] * -s; a1 += v[8] * s;
    double o = 0.0;
    o += a0 * a0;
    o += a1 * a1;
    return sqrt(o) / 1.4142135623730951;
}

template <typename T>
__global__ void __launch_bounds__(CT_THREADS)
k_ct_scharr(const SliceIn* __restrict__ in, int H, int W, double* __restrict__ E, unsigned long long* __restrict__ emax) {
    const int s = blockIdx.z, y = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
    const SliceIn si = in[s];
    double e = 0.0;
    if (x < W) {
        const T* f = (const T*)si.raw;
        double v[9], c[9];
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int i = 0; i < 3; i++) {
                const double h = hu_at(f, W, reflect1(y + j - 1, H), reflect1(x + i - 1, W), si.slope, si.intercept);
                v[j * 3 + i] = h;
                c[j * 3 + i] = fmin(fmax(h, -1000.0), 1000.0);
            }
        e = scharr3(v);
        E[((size_t)s * H + y) * W + x] = scharr3(c);
    }
    // slice maximum of the unclipped edges (>= 0, so the bit pattern orders them)
    unsigned long long k = (unsigned long long)__double_as_longlong(e);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) k = max(k, __shfl_xor_sync(0xffffffffu, k, o));
    if ((threadIdx.x & 31) == 0) atomicMax(&emax[s], k);
}

__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// threshold_otsu(S) of each slice (one CTA per slice)
__global__ void __launch_bounds__(CT_SEL_THREADS)
k_ct_otsu(const double* __restrict__ S, int HW, double* __restrict__ thres) {
    __shared__ double rmn[32], rmx[32];
    __shared__ double edge[CT_BINS + 1];
    __shared__ unsigned int hist[CT_BINS];
    __shared__ double cum_hi[CT_BINS];
    __shared__ long long w2[CT_BINS];
    const double* f = S + (size_t)blockIdx.x * HW;
    double mn = INFINITY, mx = -INFINITY;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) { const double v = f[i]; mn = fmin(mn, v); mx = fmax(mx, v); }
    mn = warp_min(mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { rmn[threadIdx.x >> 5] = mn; rmx[threadIdx.x >> 5] = mx; }
    for (int i = threadIdx.x; i < CT_BINS; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    mn = rmn[0]; mx = rmx[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) { mn = fmin(mn, rmn[k]); mx = fmax(mx, rmx[k]); }
    if (mn == mx) {                       // np.all(image == first_pixel): the threshold is that value
        if (threadIdx.x == 0) thres[blockIdx.x] = mn;
        return;
    }
    // np.linspace(mn, mx, 257): i * step + start, the last edge exactly mx
    const double step = (mx - mn) / (double)CT_BINS;
    for (int i = threadIdx.x; i <= CT_BINS; i += blockDim.x) edge[i] = i == CT_BINS ? mx : (double)i * step + mn;
    __syncthreads();
    const double denom = mx - mn;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
        const double v = f[i];
        int b = (int)(((v - mn) / denom) * (double)CT_BINS);
        if (b == CT_BINS) b--;
        if (v < edge[b]) b--;
        if (v >= edge[b + 1] && b != CT_BINS - 1) b++;
        atomicAdd(&hist[b], 1u);
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    // weight1 / weight2 (int64 cumsums), the class means from float64 cumsums of counts * centres, variance12's argmax
    double acc = 0.0;
    long long w = 0;
    for (int i = CT_BINS - 1; i >= 0; i--) {
        const double centre = (edge[i] + edge[i + 1]) / 2.0;
        acc += (double)hist[i] * centre;
        w += hist[i];
        cum_hi[i] = acc;
        w2[i] = w;
    }
    double best = -INFINITY, lo = 0.0;
    int arg = 0;
    long long w1 = 0;
    for (int i = 0; i < CT_BINS - 1; i++) {
        const double centre = (edge[i] + edge[i + 1]) / 2.0;
        lo += (double)hist[i] * centre;
        w1 += hist[i];
        const double m1 = lo / (double)w1, m2 = cum_hi[i + 1] / (double)w2[i + 1];
        const double d = m1 - m2;
        const double var = (double)(w1 * w2[i + 1]) * (d * d);
        if (var > best) { best = var; arg = i; }
    }
    thres[blockIdx.x] = (edge[arg] + edge[arg + 1]) / 2.0;
}

// The planes P and Q hold a chunk's slices one after the other, as union-find forests with slice-local parents: pixel i of the chunk
// is pixel p = i % HW of its slice, whose planes start at i - p.  A chunk has at most CT_CHUNK_PIXELS pixels, so i is an int.

__global__ void k_ct_binarize(const double* __restrict__ S, const double* __restrict__ thres, int HW, int N, int* __restrict__ P) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) P[i] = S[i] > thres[i / HW] ? i % HW : -1;
}

__global__ void k_ct_flatten(int HW, int N, int* __restrict__ P) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || P[i] < 0) return;
    const int p = i % HW;
    P[i] = ccl_root(P + (i - p), p);
}

// flag[root] = 1 for every component of P with a pixel in the band of `ext` rows / columns along the slice's border
__global__ void k_ct_mark_border(int H, int W, int N, int ext, const int* __restrict__ P, int* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || P[i] < 0) return;
    const int p = i % (H * W), y = p / W, x = p - y * W;
    if (y < ext || y >= H - ext || x < ext || x >= W - ext) flag[i - p + P[i]] = 1;
}

__global__ void k_ct_clear_flagged(int HW, int N, int* __restrict__ P, const int* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N && P[i] >= 0 && flag[i - i % HW + P[i]]) P[i] = -1;
}

// Q: the background (P < 0) as its own union-find forest
__global__ void k_ct_background(int HW, int N, const int* __restrict__ P, int* __restrict__ Q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) Q[i] = P[i] < 0 ? i % HW : -1;
}

// binary_fill_holes: a background pixel stays background when its 4-connected background component reaches the slice's edge
// (flag[root] set by k_ct_mark_border with ext = 1).  P becomes the filled mask, ready to be labelled.
__global__ void k_ct_fill(int HW, int N, int* __restrict__ P, const int* __restrict__ Q, const int* __restrict__ flag,
                          uint8_t* __restrict__ filled) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int p = i % HW;
    const bool fg = P[i] >= 0 || !flag[i - p + Q[i]];
    P[i] = fg ? p : -1;
    if (filled) filled[i] = fg ? 1 : 0;
}

__global__ void k_ct_region_sums(int H, int W, int N, const int* __restrict__ P, unsigned int* __restrict__ area,
                                 unsigned long long* __restrict__ rsum, unsigned long long* __restrict__ csum) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || P[i] < 0) return;
    const int p = i % (H * W), y = p / W, x = p - y * W;
    const int r = i - p + P[i];
    atomicAdd(&area[r], 1u);
    if (y) atomicAdd(&rsum[r], (unsigned long long)y);
    if (x) atomicAdd(&csum[r], (unsigned long long)x);
}

__device__ __forceinline__ unsigned long long block_min_u64(unsigned long long v, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long r = red[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) r = min(r, red[k]);
    return r;
}

// the phantom region of each slice and its status row (one CTA per slice)
__global__ void __launch_bounds__(CT_SEL_THREADS)
k_ct_select(int HW, const int* __restrict__ P, const unsigned int* __restrict__ area, const unsigned long long* __restrict__ rsum,
            const unsigned long long* __restrict__ csum, const unsigned long long* __restrict__ emax, const double* __restrict__ thres,
            double catphan_size, epid_ct_slice* __restrict__ rows) {
    __shared__ unsigned long long red[32];
    const int s = blockIdx.x;
    const int base = s * HW;
    unsigned long long best = ~0ull, count = 0;
    for (int p = threadIdx.x; p < HW; p += blockDim.x) {
        if (P[base + p] != p) continue;
        count++;
        const double key = fabs((double)area[base + p] - catphan_size);
        best = min(best, (unsigned long long)__double_as_longlong(key));
    }
    best = block_min_u64(best, red);
    // the first label among the best keys
    unsigned long long root = ~0ull;
    for (int p = threadIdx.x; p < HW; p += blockDim.x) {
        if (P[base + p] != p) continue;
        if ((unsigned long long)__double_as_longlong(fabs((double)area[base + p] - catphan_size)) == best) { root = p; break; }
    }
    root = block_min_u64(root, red);
    unsigned long long nreg = 0;
    for (int o = 16; o > 0; o >>= 1) count += __shfl_xor_sync(0xffffffffu, count, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = count;
    __syncthreads();
    for (int k = 0; k < (int)(blockDim.x >> 5); k++) nreg += red[k];
    if (threadIdx.x != 0) return;
    epid_ct_slice& r = rows[s];
    r.max_edge = __longlong_as_double((long long)emax[s]);
    r.threshold = thres[s];
    r.n_regions = r.max_edge >= 0.1 ? (int32_t)nreg : 0;    // the reference stops at the edge check
    r.label = -1;
    r.area = 0;
    r.centroid_row = r.centroid_col = NAN;
    if (!(r.max_edge >= 0.1)) {
        r.status = EPID_CT_NO_EDGES;
    } else if (nreg < 1) {
        r.status = EPID_CT_NO_REGIONS;
    } else {
        const int g = base + (int)root;
        const double a = (double)area[g];
        r.label = (int32_t)root;
        r.area = (int32_t)area[g];
        r.centroid_row = (double)rsum[g] / a;
        r.centroid_col = (double)csum[g] / a;
        const bool too_large = catphan_size * 1.3 < a, too_small = a < catphan_size / 1.3;
        r.status = (too_large || too_small) ? EPID_CT_WRONG_SIZE : EPID_CT_OK;
    }
}

inline unsigned blocks(int N) { return (unsigned)((N + CT_THREADS - 1) / CT_THREADS); }

template <class T>
int launch_scharr(epid_ctx* ctx, const SliceIn* d_in, int m, int H, int W, double* E, unsigned long long* emax) {
    k_ct_scharr<T><<<dim3((W + CT_THREADS - 1) / CT_THREADS, H, m), CT_THREADS, 0, ctx->stream>>>(d_in, H, W, E, emax);
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_ct_localize(epid_ctx* ctx, const epid_batch* volume, const double* slope, const double* intercept,
                                    const int32_t* slices, int32_t nslices, double catphan_size, int32_t clear_borders,
                                    int32_t clip_in_localization, const double* gauss_w, int32_t gauss_r, struct epid_ct_slice* results,
                                    double* scharr, double* smoothed, uint8_t* filled, int32_t* labels) {
    EPID_REQUIRE(ctx && volume && slope && intercept && slices && results && gauss_w, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(clip_in_localization, EPID_ERR_UNSUPPORTED,
                 "localization without clipping (a Slice passed to get_regions) is not implemented");
    EPID_REQUIRE(volume->dtype == EPID_I16 || volume->dtype == EPID_U16, EPID_ERR_UNSUPPORTED,
                 "CT localization reads int16 or uint16 slices");
    EPID_REQUIRE(nslices >= 0 && gauss_r >= 0, EPID_ERR_INVALID, "bad slice count or Gaussian radius");
    const int H = volume->h, W = volume->w;
    // the kernels put a slice's rows in grid.y
    EPID_REQUIRE(H >= 2 && W >= 2 && H <= CT_MAX_GRID && (long long)H * W <= CT_CHUNK_PIXELS, EPID_ERR_UNSUPPORTED,
                 "slices of %d x %d pixels are not supported (at least 2 x 2, at most %d rows and %lld pixels)", H, W, CT_MAX_GRID,
                 CT_CHUNK_PIXELS);
    // clear_border's band: buffer_size = min(int(max(H, W) / 100), 3) rows / columns plus one
    const int ext = std::min((int)((double)std::max(H, W) / 100.0), 3) + 1;
    EPID_REQUIRE(!clear_borders || (ext - 1 < H && ext - 1 < W), EPID_ERR_INVALID, "buffer size may not be greater than labels size");
    for (int k = 0; k < nslices; k++)
        EPID_REQUIRE(slices[k] >= 0 && slices[k] < volume->n, EPID_ERR_INVALID, "slice %d is outside the series of %d", slices[k], volume->n);
    if (nslices == 0) return EPID_OK;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const long long HW = (long long)H * W;
    // a chunk's slices go in grid.z
    const int chunk = (int)std::min<long long>(std::min<long long>(nslices, CT_CHUNK_PIXELS / HW), CT_MAX_GRID);
    const long long NC = HW * chunk;
    const size_t esz = dtype_size(volume->dtype);

    // one allocation: per-slice inputs, edge maxima, thresholds, rows; then the planes of one chunk
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
    const size_t o_in = take(sizeof(SliceIn) * chunk), o_emax = take(8 * chunk), o_thr = take(8 * chunk), o_rows = take(sizeof(epid_ct_slice) * chunk);
    const size_t o_E = take(8 * NC), o_T = take(8 * NC), o_S = take(8 * NC), o_P = take(4 * NC), o_Q = take(4 * NC), o_A = take(4 * NC);
    const size_t o_R = take(8 * NC), o_C = take(8 * NC), o_F = take(NC);
    char* d = nullptr;
    EPID_CUDA(cudaMallocAsync((void**)&d, off, ctx->stream));
    SliceIn* d_in = (SliceIn*)(d + o_in);
    unsigned long long* d_emax = (unsigned long long*)(d + o_emax);
    double* d_thr = (double*)(d + o_thr);
    epid_ct_slice* d_rows = (epid_ct_slice*)(d + o_rows);
    double *E = (double*)(d + o_E), *T = (double*)(d + o_T), *S = (double*)(d + o_S);
    int *P = (int*)(d + o_P), *Q = (int*)(d + o_Q), *flag = (int*)(d + o_A);
    unsigned int* A = (unsigned int*)(d + o_A);
    unsigned long long *R = (unsigned long long*)(d + o_R), *Cs = (unsigned long long*)(d + o_C);
    uint8_t* F = (uint8_t*)(d + o_F);

    std::vector<SliceIn> hin(chunk);
    cudaError_t e = cudaSuccess;
    int rc = EPID_OK;
    for (int k0 = 0; k0 < nslices && rc == EPID_OK && e == cudaSuccess; k0 += chunk) {
        const int m = std::min(chunk, nslices - k0);
        const int N = (int)(HW * m);
        const dim3 g_union(blocks((int)HW), m);      // one thread per pixel, slices in grid.y
        for (int j = 0; j < m; j++) {
            const int sl = slices[k0 + j];
            hin[j] = SliceIn{(const char*)volume->dptr + (size_t)sl * HW * esz, slope[sl], intercept[sl]};
        }
        // the inputs are staged from host memory that changes per chunk: copy synchronously with respect to the host
        e = cudaMemcpyAsync(d_in, hin.data(), sizeof(SliceIn) * m, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_emax, 0, 8 * m, ctx->stream);
        if (e != cudaSuccess) break;
        rc = volume->dtype == EPID_I16 ? launch_scharr<int16_t>(ctx, d_in, m, H, W, E, d_emax) : launch_scharr<uint16_t>(ctx, d_in, m, H, W, E, d_emax);
        if (rc == EPID_OK) rc = correlate1d_f64(ctx, E, T, m, H, W, 0, gauss_w, gauss_r, 1);
        if (rc == EPID_OK) rc = correlate1d_f64(ctx, T, S, m, H, W, 1, gauss_w, gauss_r, 1);
        if (rc != EPID_OK) break;
        k_ct_otsu<<<m, CT_SEL_THREADS, 0, ctx->stream>>>(S, (int)HW, d_thr);
        k_ct_binarize<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(S, d_thr, (int)HW, N, P);
        if (clear_borders) {
            k_ccl_union<<<g_union, CT_THREADS, 0, ctx->stream>>>(H, W, 1, P);
            k_ct_flatten<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, P);
            e = cudaMemsetAsync(flag, 0, 4 * N, ctx->stream);
            if (e != cudaSuccess) break;
            k_ct_mark_border<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(H, W, N, ext, P, flag);
            k_ct_clear_flagged<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, P, flag);
        }
        k_ct_background<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, P, Q);
        k_ccl_union<<<g_union, CT_THREADS, 0, ctx->stream>>>(H, W, 0, Q);
        k_ct_flatten<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, Q);
        e = cudaMemsetAsync(flag, 0, 4 * N, ctx->stream);
        if (e != cudaSuccess) break;
        k_ct_mark_border<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(H, W, N, 1, Q, flag);
        k_ct_fill<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, P, Q, flag, F);
        k_ccl_union<<<g_union, CT_THREADS, 0, ctx->stream>>>(H, W, 1, P);
        k_ct_flatten<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, P);
        e = cudaMemsetAsync(A, 0, 4 * N, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(R, 0, 8 * N, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(Cs, 0, 8 * N, ctx->stream);
        if (e != cudaSuccess) break;
        k_ct_region_sums<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(H, W, N, P, A, R, Cs);
        k_ct_select<<<m, CT_SEL_THREADS, 0, ctx->stream>>>((int)HW, P, A, R, Cs, d_emax, d_thr, catphan_size, d_rows);
        ctx->launches += clear_borders ? 16 : 12;
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(results + k0, d_rows, sizeof(epid_ct_slice) * m, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && scharr) e = cudaMemcpyAsync(scharr + HW * k0, E, 8 * N, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && smoothed) e = cudaMemcpyAsync(smoothed + HW * k0, S, 8 * N, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && filled) e = cudaMemcpyAsync(filled + HW * k0, F, N, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && labels) e = cudaMemcpyAsync(labels + HW * k0, P, 4 * N, cudaMemcpyDeviceToHost, ctx->stream);
        // hin is rewritten by the next chunk: wait for this one
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    }
    const cudaError_t ef = cudaFreeAsync(d, ctx->stream);
    if (e == cudaSuccess) e = ef;
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (rc != EPID_OK) return rc;
    if (e != cudaSuccess) {
        set_error("epid_ct_localize failed: %s", cudaGetErrorString(e));
        return EPID_ERR_CUDA;
    }
    return EPID_OK;
}
