// pylinac.nuclear.TomographicUniformity (nuclear.py:1370-1551) on the device: the slab mean of a SPECT volume and PlanarUniformity's
// pipeline on that float64 frame, bit-identical to the reference.
//
//   k_tu_bin    streaming stage, one CTA per (binned row, volume): the exact integer sum T of the slab's `count` slices per raw pixel,
//               the mean m = T / count (one rounding, as numpy's mean(axis=0)), and the block sums of m to the bin, the bottom / right
//               edges zero-padded: per block acc = 0; acc += pw(row) for each of its rows (skimage's block_reduce(func=np.sum)).
//   k_tu_frame  one CTA per volume on the float64 binned frame, held in shared memory when 16 bytes per pixel fit (the global
//               workspace otherwise; same code): convolve2d's order for the 9-point filter, edge zeroing, the threshold (the values
//               above 10 % of the max compacted in raster order and their pairwise-sum mean), then the stray-pixel stencil and the
//               stages of nuclear_stages.cuh shared with k_nm_frame for three FOVs (UFOV, CFOV, center), and the center and ring sums of
//               center_border_ratio as pairwise sums over the whole frame.
//
// Exactness (DESIGN.md section 4.16): the mean frame is not integer, so every sum rounds; each is evaluated in numpy's or scipy's own
// order (np_sum.cuh, -fmad=false), and everything after the threshold is decided on value > 0.
#include "common.cuh"
#include "np_sum.cuh"
#include "nuclear_stages.cuh"

#include <cmath>

namespace epid {
namespace {

using namespace nm;

constexpr int TU_BIN_THREADS = 256;
constexpr int TU_TILE = 4096;          // doubles of k_tu_bin's mean tile: bin raw rows x TU_TILE / bin raw columns
constexpr int TU_THREADS = 512;
constexpr int TU_LOG_THREADS = 9;
constexpr size_t TU_STATIC_SMEM = 8192;   // red[], wsum[] and slots[] of k_tu_frame, rounded up

__global__ void __launch_bounds__(TU_BIN_THREADS) k_tu_bin(const uint16_t* __restrict__ vol, int nz, int h, int w, int first, int count,
                                                           int bin, int hb, int wb, double* __restrict__ binned, double* __restrict__ mean) {
    __shared__ double tile[TU_TILE];
    const int i = blockIdx.x, v = blockIdx.y;
    const size_t plane = (size_t)h * w;
    const uint16_t* src = vol + ((size_t)v * nz + first) * plane;
    const int cols = TU_TILE / bin;    // a multiple of the bin
    const int r0 = i * bin;
    double* dst = binned + ((size_t)v * hb + i) * wb;
    for (int c0 = 0; c0 < wb * bin; c0 += cols) {
        const int ncols = min(cols, wb * bin - c0);
        for (int e = threadIdx.x; e < bin * ncols; e += TU_BIN_THREADS) {
            const int rr = e / ncols, c = e - rr * ncols;
            const int row = r0 + rr, col = c0 + c;
            double m = 0.0;
            if (row < h && col < w) {
                const uint16_t* q = src + (size_t)row * w + col;
                unsigned long long t = 0;
                int s = 0;
                for (; s + 4 <= count; s += 4)
                    t += (uint32_t)q[(size_t)s * plane] + q[(size_t)(s + 1) * plane] + q[(size_t)(s + 2) * plane] +
                         q[(size_t)(s + 3) * plane];
                for (; s < count; s++) t += q[(size_t)s * plane];
                m = (double)t / (double)count;
                if (mean) mean[(size_t)v * plane + (size_t)row * w + col] = m;
            }
            tile[rr * cols + c] = m;
        }
        __syncthreads();
        for (int jj = threadIdx.x; jj < ncols / bin; jj += TU_BIN_THREADS) {
            double acc = 0.0;
            for (int rr = 0; rr < bin; rr++) {                 // bin <= 64: every row is one pairwise leaf
                const double* rowp = tile + rr * cols + jj * bin;
                acc += np::pw_leaf([&](long long k) { return rowp[k]; }, 0, bin);
            }
            dst[c0 / bin + jj] = acc;
        }
        __syncthreads();
    }
}

struct TuPlanes {                 // optional device outputs of k_tu_frame (nullptr: not written)
    double* filtered;             // [n][hb][wb] after the filter and edge zeroing
    double* cleaned;              // [n][hb][wb] after the threshold and the stray-pixel stencil (the reference's binned_frame)
    int32_t* edt2;                // [n][hb][wb] squared distance to the nearest background pixel
    uint8_t* masks;               // [n][3][hb][wb] UFOV, CFOV and center masks
};

__global__ void __launch_bounds__(TU_THREADS) k_tu_frame(const double* __restrict__ binned, int hb, int wb, double ufov_erode,
                                                         double cfov_erode, double center_erode, int win, double thr_frac, double* ws,
                                                         epid_tu_result* res, TuPlanes out) {
    extern __shared__ __align__(16) double tsm[];
    __shared__ unsigned long long red[32];
    __shared__ int wsum[32];
    __shared__ double slots[TU_THREADS];
    const int f = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int N = hb * wb;
    const size_t fo = (size_t)f * N;
    double* M = ws ? ws + 2 * fo : tsm;
    int* P = (int*)(M + N);       // -1 / union-find parent; later the squared EDT
    int* A = P + N;               // component areas; later the column distances of the EDT
    double* SEL = (double*)P;     // the threshold selection in raster order, before the stencil
    const double* B = binned + fo;
    epid_tu_result r = {};

    // ---- convolve2d(B, [[1,2,1],[2,4,2],[1,2,1]] / 16, "same"): from 0, rows +1, 0, -1, each column +1, 0, -1; outer rows / columns 0
    unsigned long long mkey = 0;
    for (int p = tid; p < N; p += nt) {
        const int i = p / wb, j = p - i * wb;
        double s = 0.0;
        if (i > 0 && i < hb - 1 && j > 0 && j < wb - 1) {
            const double* q = B + p;
            s += q[wb + 1] * 0.0625;
            s += q[wb] * 0.125;
            s += q[wb - 1] * 0.0625;
            s += q[1] * 0.125;
            s += q[0] * 0.25;
            s += q[-1] * 0.125;
            s += q[-wb + 1] * 0.0625;
            s += q[-wb] * 0.125;
            s += q[-wb - 1] * 0.0625;
        }
        M[p] = s;
        mkey = max(mkey, value_key(s));
        if (out.filtered) out.filtered[fo + p] = s;
    }
    // ---- threshold: array[array > max * 0.10].mean() * thr_frac, the selection compacted in raster order (contiguous runs per thread)
    const double t10 = __longlong_as_double((long long)block_reduce(mkey, OpMax(), red)) * 0.10;
    const int run = (N + nt - 1) / nt, p0 = min(N, tid * run), p1 = min(N, p0 + run);
    int c = 0;
    for (int p = p0; p < p1; p++) c += M[p] > t10;
    int incl = c;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if ((tid & 31) >= o) incl += y;
    }
    if ((tid & 31) == 31) wsum[tid >> 5] = incl;
    __syncthreads();
    int off = incl - c, total = 0;
    for (int k = 0; k < nt / 32; k++) {
        if (k < (tid >> 5)) off += wsum[k];
        total += wsum[k];
    }
    for (int p = p0; p < p1; p++)
        if (M[p] > t10) SEL[off++] = M[p];
    __syncthreads();
    const double sel_sum = np::block_pw([&](long long k) { return SEL[k]; }, total, TU_LOG_THREADS, slots);
    const double thr = total ? (0.0 + sel_sum) / (double)total * thr_frac : NAN;   // the mean of an empty selection is nan
    r.threshold = thr;
    for (int p = tid; p < N; p += nt)
        if (M[p] < thr) M[p] = 0.0;
    __syncthreads();
    remove_stray_pixels(M, P, hb, wb, [&](int p, double m) {
        if (out.cleaned) out.cleaned[fo + p] = m;
    });

    label_areas(P, A, hb, wb);
    const int longest = largest_component(P, A, hb, wb, red).longest;
    if (longest == 0) {           // no component: get_fov's max() over no regions raises
        if (tid == 0) {
            r.status = EPID_NM_NO_COMPONENT;
            res[f] = r;
        }
        return;
    }
    // int(round((1 - size) * longest)): Python rounds halves to even, as rint does
    r.longest = longest;
    r.erosion[0] = (int)rint(ufov_erode * (double)longest);
    r.erosion[1] = (int)rint(cfov_erode * (double)longest);
    r.erosion[2] = (int)rint(center_erode * (double)longest);
    squared_edt(P, A, hb, wb, out.edt2 ? out.edt2 + fo : nullptr);
    const FovMasks<3> in_fov(r.erosion);
    fov_uniformity<3>(M, P, in_fov, hb, wb, win, out.masks ? out.masks + 3 * fo : nullptr, red, r);

    // ---- center_border_ratio: np.nanmean of the center FOV and of the ring (UFOV without the CFOV), zeros as nan: each sum is
    // np.sum of the whole frame with zeros outside the set
    auto center = [&](long long p) { return in_fov(P, (int)p, 2) && M[p] > 0 ? M[p] : 0.0; };
    auto ring = [&](long long p) { return in_fov(P, (int)p, 0) && M[p] > 0 && !in_fov(P, (int)p, 1) ? M[p] : 0.0; };
    r.center_sum = 0.0 + np::block_pw(center, N, TU_LOG_THREADS, slots);
    r.ring_sum = 0.0 + np::block_pw(ring, N, TU_LOG_THREADS, slots);
    unsigned long long nc = 0, nr = 0;
    for (int p = tid; p < N; p += nt) {
        nc += center(p) > 0;
        nr += ring(p) > 0;
    }
    r.center_count = (int)block_reduce(nc, OpSum(), red);
    r.ring_count = (int)block_reduce(nr, OpSum(), red);
    if (tid == 0) res[f] = r;
}

// ctx->scratch: [binned frames] [result rows] [per-volume workspace when the frame does not fit shared memory] [extra]
int tu_scratch(epid_ctx* ctx, int nvol, int hb, int wb, size_t extra, FrameScratch* s) {
    const size_t N = (size_t)hb * wb;
    return frame_scratch(ctx, nvol, N, 16, TU_STATIC_SMEM, 8 * N * nvol, nvol * sizeof(epid_tu_result), extra, s);
}

int tu_check(const epid_batch* volumes, int nz, int first, int count, int bin, int window, int* hb, int* wb) {
    int rc = check_volumes(volumes, nz, "tomographic volumes");
    if (rc != EPID_OK) return rc;
    EPID_REQUIRE(first >= 0 && count >= 1 && (long long)first + count <= nz, EPID_ERR_INVALID, "slab [%d, %d + %d) of %d slices", first,
                 first, count, nz);
    return check_binning(volumes, bin, window, 1LL << 28, hb, wb);
}

int tu_launch(epid_ctx* ctx, const epid_batch* volumes, int nz, int first, int count, int bin, const double* erode, int window,
              double thr, const FrameScratch& s, int hb, int wb, double* mean, const TuPlanes& planes) {
    const int nvol = volumes->n / nz;
    double* binned = (double*)s.head;
    k_tu_bin<<<dim3(hb, nvol), TU_BIN_THREADS, 0, ctx->stream>>>((const uint16_t*)volumes->dptr, nz, volumes->h, volumes->w, first, count,
                                                                  bin, hb, wb, binned, mean);
    EPID_CUDA(cudaGetLastError());
    EPID_SMEM_OPT_IN(ctx, k_tu_frame, s.smem);
    k_tu_frame<<<nvol, TU_THREADS, s.smem, ctx->stream>>>(binned, hb, wb, erode[0], erode[1], erode[2], window, thr, (double*)s.ws,
                                                          (epid_tu_result*)s.rows, planes);
    EPID_CUDA(cudaGetLastError());
    ctx->launches += 2;
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_tu_uniformity(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, int32_t first, int32_t count, int32_t bin,
                                      double ufov_erode, double cfov_erode, double center_erode, int32_t window, double threshold,
                                      struct epid_tu_result* results, epid_batch** mean, epid_batch** cleaned, epid_batch** masks) {
    EPID_REQUIRE(ctx && results, EPID_ERR_INVALID, "NULL argument");
    int hb, wb;
    int rc = tu_check(volumes, nz, first, count, bin, window, &hb, &wb);
    if (rc != EPID_OK) return rc;
    const int nvol = volumes->n / nz;
    if (nvol == 0) return EPID_OK;
    EPID_CUDA(cudaSetDevice(ctx->device));
    FrameScratch s;
    if ((rc = tu_scratch(ctx, nvol, hb, wb, 0, &s)) != EPID_OK) return rc;
    TuPlanes planes = {};
    epid_batch *bmean = nullptr, *bc = nullptr, *bm = nullptr;
    auto release = [&]() {
        epid_batch_free(bmean);
        epid_batch_free(bc);
        epid_batch_free(bm);
    };
    if (mean && (rc = epid_batch_alloc(ctx, EPID_F64, nvol, volumes->h, volumes->w, &bmean)) != EPID_OK) return rc;
    if (cleaned && (rc = epid_batch_alloc(ctx, EPID_F64, nvol, hb, wb, &bc)) != EPID_OK) {
        release();
        return rc;
    }
    if (masks && (rc = epid_batch_alloc(ctx, EPID_U8, 3 * nvol, hb, wb, &bm)) != EPID_OK) {
        release();
        return rc;
    }
    if (bc) planes.cleaned = (double*)bc->dptr;
    if (bm) planes.masks = (uint8_t*)bm->dptr;
    const double erode[3] = {ufov_erode, cfov_erode, center_erode};
    rc = tu_launch(ctx, volumes, nz, first, count, bin, erode, window, threshold, s, hb, wb, bmean ? (double*)bmean->dptr : nullptr, planes);
    if (rc == EPID_OK) rc = finish(ctx, results, s.rows, nvol * sizeof(epid_tu_result), "tomographic uniformity");
    if (rc != EPID_OK) {
        cudaStreamSynchronize(ctx->stream);   // k_tu_bin may still be writing the slab means when k_tu_frame failed to launch
        release();
        return rc;
    }
    if (mean) *mean = bmean;
    if (cleaned) *cleaned = bc;
    if (masks) *masks = bm;
    return EPID_OK;
}

extern "C" int32_t epid_tu_stages(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, int32_t first, int32_t count, int32_t bin,
                                  double ufov_erode, double cfov_erode, double center_erode, int32_t window, double threshold,
                                  struct epid_tu_result* results, double* mean, double* binned, double* filtered, double* cleaned,
                                  int32_t* edt2, uint8_t* masks) {
    EPID_REQUIRE(ctx && results && mean && binned && filtered && cleaned && edt2 && masks, EPID_ERR_INVALID, "NULL argument");
    int hb, wb;
    int rc = tu_check(volumes, nz, first, count, bin, window, &hb, &wb);
    if (rc != EPID_OK) return rc;
    const int nvol = volumes->n / nz;
    if (nvol == 0) return EPID_OK;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t plane = (size_t)nvol * hb * wb, raw = (size_t)nvol * volumes->h * volumes->w;
    const size_t b8 = align256(8 * plane), b4 = align256(4 * plane), b_mean = align256(8 * raw);
    FrameScratch s;
    if ((rc = tu_scratch(ctx, nvol, hb, wb, b_mean + 2 * b8 + b4 + align256(3 * plane), &s)) != EPID_OK) return rc;
    double* dmean = (double*)s.extra;
    TuPlanes planes = {};
    planes.filtered = (double*)(s.extra + b_mean);
    planes.cleaned = (double*)(s.extra + b_mean + b8);
    planes.edt2 = (int32_t*)(s.extra + b_mean + 2 * b8);
    planes.masks = (uint8_t*)(s.extra + b_mean + 2 * b8 + b4);
    EPID_CUDA(cudaMemsetAsync(planes.edt2, 0xff, 4 * plane, ctx->stream));    // -1 where a frame stops before its EDT
    EPID_CUDA(cudaMemsetAsync(planes.masks, 0, 3 * plane, ctx->stream));
    const double erode[3] = {ufov_erode, cfov_erode, center_erode};
    if ((rc = tu_launch(ctx, volumes, nz, first, count, bin, erode, window, threshold, s, hb, wb, dmean, planes)) != EPID_OK) return rc;
    EPID_CUDA(cudaMemcpyAsync(results, s.rows, nvol * sizeof(epid_tu_result), cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(mean, dmean, 8 * raw, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(binned, s.head, 8 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(filtered, planes.filtered, 8 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(cleaned, planes.cleaned, 8 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(edt2, planes.edt2, 4 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(masks, planes.masks, 3 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    return EPID_OK;
}
