// pylinac.nuclear.PlanarUniformity (nuclear.py:151-500) on the device: NEMA integral and differential uniformity of gamma-camera
// flood frames, bit-identical to the reference.
//
//   k_nm_bin    streaming stage, one CTA per (binned row, frame): the raw uint16 frame -> exact uint32 block sums of bin x bin pixels,
//               the bottom / right edges zero-padded up to a multiple of the bin (skimage block_reduce(func=np.sum)).
//   k_nm_frame  one CTA per frame on the binned frame, held in shared memory when 12 bytes per binned pixel fit (the global workspace
//               otherwise; same code): the 9-point filter as the exact integer S = 16 x filtered value, edge zeroing, threshold,
//               stray-pixel stencil, 4-connected labelling with the largest component's area and bounding box, one exact squared EDT,
//               both FOV masks, integral uniformity with its max / min points and differential uniformity with its argmax per axis.
//
// Exactness (DESIGN.md section 4.14): every filtered value is S / 16 with S an integer, so the threshold mean, the Michelson ratios
// and the EDT comparison are evaluated on exact integers and round once, as numpy does.
#include "ccl.cuh"
#include "common.cuh"
#include "nuclear_stages.cuh"

#include <climits>
#include <cmath>

namespace epid {
namespace {

using namespace nm;

constexpr int NM_BIN_THREADS = 256;
constexpr int NM_BIN_COLS = 2048;      // raw columns per pass of k_nm_bin (a multiple of every supported bin)
constexpr int NM_THREADS = 512;
constexpr int NM_MAX_BIN = 64;         // 16 * 65535 * 64^2 < 2^32: S stays a uint32

// block sums of bin x bin raw pixels for binned row blockIdx.x of frame blockIdx.y.  Each thread sums raw columns over the bin's rows
// (coalesced along the row), then each binned column adds its bin column sums.  VEC: w % 8 == 0, 16-byte loads of 8 pixels.
template <bool VEC>
__global__ void __launch_bounds__(NM_BIN_THREADS) k_nm_bin(const uint16_t* __restrict__ raw, int h, int w, int bin, int hb, int wb,
                                                           uint32_t* __restrict__ binned) {
    __shared__ uint32_t colsum[NM_BIN_COLS];
    const int i = blockIdx.x;
    const uint16_t* src = raw + (size_t)blockIdx.y * h * w;
    const int r0 = i * bin, r1 = min(r0 + bin, h);
    uint32_t* dst = binned + ((size_t)blockIdx.y * hb + i) * wb;
    for (int c0 = 0; c0 < wb * bin; c0 += NM_BIN_COLS) {
        const int ncols = min(NM_BIN_COLS, wb * bin - c0);
        if (VEC) {
            for (int c = threadIdx.x * 8; c < ncols; c += NM_BIN_THREADS * 8) {
                uint32_t s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                if (c0 + c < w) {                           // w and c0 + c are multiples of 8: all 8 columns are inside
                    for (int r = r0; r < r1; r++) {
                        const uint4 v = ldg_stream16(src + (size_t)r * w + c0 + c);
                        s[0] += v.x & 0xffffu; s[1] += v.x >> 16; s[2] += v.y & 0xffffu; s[3] += v.y >> 16;
                        s[4] += v.z & 0xffffu; s[5] += v.z >> 16; s[6] += v.w & 0xffffu; s[7] += v.w >> 16;
                    }
                }
#pragma unroll
                for (int k = 0; k < 8; k++) colsum[c + k] = s[k];
            }
        } else {
            for (int c = threadIdx.x; c < ncols; c += NM_BIN_THREADS) {
                uint32_t s = 0;
                if (c0 + c < w)
                    for (int r = r0; r < r1; r++) s += src[(size_t)r * w + c0 + c];
                colsum[c] = s;
            }
        }
        __syncthreads();
        for (int jj = threadIdx.x; jj < ncols / bin; jj += NM_BIN_THREADS) {
            uint32_t s = 0;
            for (int k = 0; k < bin; k++) s += colsum[jj * bin + k];
            dst[c0 / bin + jj] = s;
        }
        __syncthreads();
    }
}

struct NmPlanes {                 // optional device outputs of k_nm_frame (nullptr: not written)
    double* cleaned;              // [n][hb][wb] cleaned frame S / 16 (the reference's binned_frame)
    uint8_t* masks;               // [n][2][hb][wb] UFOV, CFOV masks (the reference's eroded binary)
    uint32_t* filtered;           // [n][hb][wb] S after the filter and edge zeroing
    uint32_t* clean_s;            // [n][hb][wb] S after the threshold and the stray-pixel stencil
    int32_t* edt2;                // [n][hb][wb] squared distance to the nearest background pixel
};

// FULL: `in` holds block sums and the frame is filtered, thresholded and cleaned first.  !FULL (get_fov): `in` is the frame's binary.
template <typename TIn, bool FULL>
__global__ void __launch_bounds__(NM_THREADS) k_nm_frame(const TIn* __restrict__ in, int hb, int wb, double ufov_erode, double cfov_erode,
                                                         int win, double thr_frac, int use_smem, uint32_t* ws, epid_nm_result* res,
                                                         NmPlanes out) {
    extern __shared__ __align__(16) uint32_t dsm[];
    __shared__ unsigned long long red[32];
    const int f = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int N = hb * wb;
    const size_t fo = (size_t)f * N;
    uint32_t* S = use_smem ? dsm : ws + 3 * fo;
    int* P = (int*)(S + N);       // -1 / union-find parent; later the squared EDT
    int* A = (int*)(S + 2 * N);   // component areas; later the column distances of the EDT
    const TIn* B = in + fo;
    epid_nm_result r = {};

    // ---- filter: S = [[1,2,1],[2,4,2],[1,2,1]] (x) binned, zero fill; the outer rows and columns are zeroed anyway
    unsigned long long smax = 0;
    for (int p = tid; p < N; p += nt) {
        const int i = p / wb, j = p - i * wb;
        uint32_t s;
        if (FULL) {
            s = 0;
            if (i > 0 && i < hb - 1 && j > 0 && j < wb - 1) {
                const TIn* q = B + p;
                s = q[-wb - 1] + 2 * q[-wb] + q[-wb + 1] + 2 * q[-1] + 4 * q[0] + 2 * q[1] + q[wb - 1] + 2 * q[wb] + q[wb + 1];
            }
            smax = s > smax ? s : smax;
            if (out.filtered) out.filtered[fo + p] = s;
        } else {
            s = B[p] != 0;
        }
        S[p] = s;
    }
    if (FULL) {
        // ---- threshold: mean of the values above 10 % of the max, times thr_frac; values below it are zeroed
        smax = block_reduce(smax, OpMax(), red);
        const double t10 = (double)smax * 0.0625 * 0.1;
        unsigned long long sum = 0, cnt = 0;
        for (int p = tid; p < N; p += nt) {
            if ((double)S[p] * 0.0625 > t10) {
                sum += S[p];
                cnt++;
            }
        }
        sum = block_reduce(sum, OpSum(), red);
        cnt = block_reduce(cnt, OpSum(), red);
        const double thr = cnt ? (double)sum * 0.0625 / (double)cnt * thr_frac : NAN;   // the mean of an empty selection is nan
        r.threshold = thr;
        for (int p = tid; p < N; p += nt)
            if ((double)S[p] * 0.0625 < thr) S[p] = 0;
        __syncthreads();
        // ---- remove_small_objects(min_size=2), connectivity 1: a foreground pixel without a 4-neighbour in the foreground goes
        for (int p = tid; p < N; p += nt) {
            const int i = p / wb, j = p - i * wb;
            const bool nb = (i > 0 && S[p - wb]) || (i < hb - 1 && S[p + wb]) || (j > 0 && S[p - 1]) || (j < wb - 1 && S[p + 1]);
            P[p] = S[p] && nb ? p : -1;
        }
        __syncthreads();
        for (int p = tid; p < N; p += nt) {
            if (P[p] < 0) S[p] = 0;
            if (out.clean_s) out.clean_s[fo + p] = S[p];
            if (out.cleaned) out.cleaned[fo + p] = (double)S[p] * 0.0625;
        }
    } else {
        __syncthreads();
        for (int p = tid; p < N; p += nt) P[p] = S[p] ? p : -1;
    }
    __syncthreads();

    label_areas(P, A, hb, wb);
    const int longest = largest_longest(P, A, hb, wb, red);
    if (longest == 0) {           // no component: get_fov's max() over no regions raises
        if (tid == 0) {
            r.status = EPID_NM_NO_COMPONENT;
            res[f] = r;
        }
        return;
    }
    // int(round((1 - size) * longest)): Python rounds halves to even, as rint does
    const int eu = (int)rint(ufov_erode * (double)longest), ec = (int)rint(cfov_erode * (double)longest);
    r.longest = longest;
    r.erosion[0] = eu;
    r.erosion[1] = ec;
    squared_edt(P, A, hb, wb, out.edt2 ? out.edt2 + fo : nullptr);
    fov_uniformity<2>(S, P, FovMasks<2>(r.erosion), hb, wb, win, out.masks ? out.masks + 2 * fo : nullptr, red, r);
    if (tid == 0) res[f] = r;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct NmScratch {
    uint32_t* binned = nullptr;
    epid_nm_result* res = nullptr;
    uint32_t* ws = nullptr;
    int use_smem = 0;
    size_t smem = 0;
};

// lays out ctx->scratch: [binned sums (full)] [result rows] [per-frame workspace when the frame does not fit shared memory] [extra]
int nm_scratch(epid_ctx* ctx, int n, int hb, int wb, bool full, size_t extra, NmScratch* s, char** extra_ptr) {
    const size_t N = (size_t)hb * wb;
    int optin = 0;
    EPID_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    s->smem = 12 * N;
    s->use_smem = s->smem + 1024 <= (size_t)optin;
    const size_t b_bin = full ? align256(N * n * sizeof(uint32_t)) : 0;
    const size_t b_res = align256(n * sizeof(epid_nm_result));
    const size_t b_ws = s->use_smem ? 0 : align256(12 * N * n);
    int rc = ensure_scratch(ctx, b_bin + b_res + b_ws + extra);
    if (rc != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    s->binned = full ? (uint32_t*)base : nullptr;
    s->res = (epid_nm_result*)(base + b_bin);
    s->ws = s->use_smem ? nullptr : (uint32_t*)(base + b_bin + b_res);
    if (extra_ptr) *extra_ptr = base + b_bin + b_res + b_ws;
    if (!s->use_smem) s->smem = 0;
    return EPID_OK;
}

int nm_check(const epid_batch* frames, int bin, int window, int* hb, int* wb) {
    EPID_REQUIRE(frames, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(frames->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "nuclear frames must be uint16 (dtype %d)", frames->dtype);
    EPID_REQUIRE(bin >= 1 && bin <= NM_MAX_BIN && (bin & (bin - 1)) == 0, EPID_ERR_UNSUPPORTED,
                 "bin size %d: expected a power of two up to %d", bin, NM_MAX_BIN);
    EPID_REQUIRE(window >= 1, EPID_ERR_INVALID, "window size %d < 1", window);
    *hb = (frames->h + bin - 1) / bin;
    *wb = (frames->w + bin - 1) / bin;
    EPID_REQUIRE((long long)*hb * *wb < (1LL << 30), EPID_ERR_UNSUPPORTED, "binned frame %d x %d is too large", *hb, *wb);
    return EPID_OK;
}

int nm_launch(epid_ctx* ctx, const epid_batch* frames, int bin, double ue, double ce, int window, double thr, const NmScratch& s, int hb,
              int wb, const NmPlanes& planes) {
    const int n = frames->n;
    const dim3 bgrid(hb, n);
    if (frames->w % 8 == 0)
        k_nm_bin<true><<<bgrid, NM_BIN_THREADS, 0, ctx->stream>>>((const uint16_t*)frames->dptr, frames->h, frames->w, bin, hb, wb, s.binned);
    else
        k_nm_bin<false><<<bgrid, NM_BIN_THREADS, 0, ctx->stream>>>((const uint16_t*)frames->dptr, frames->h, frames->w, bin, hb, wb, s.binned);
    EPID_CUDA(cudaGetLastError());
    EPID_SMEM_OPT_IN(ctx, (k_nm_frame<uint32_t, true>), s.smem);
    k_nm_frame<uint32_t, true><<<n, NM_THREADS, s.smem, ctx->stream>>>(s.binned, hb, wb, ue, ce, window, thr, s.use_smem, s.ws, s.res, planes);
    EPID_CUDA(cudaGetLastError());
    ctx->launches += 2;
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_nm_uniformity(epid_ctx* ctx, const epid_batch* frames, int32_t bin, double ufov_erode, double cfov_erode,
                                      int32_t window, double threshold, struct epid_nm_result* results, epid_batch** cleaned,
                                      epid_batch** masks) {
    EPID_REQUIRE(ctx && results, EPID_ERR_INVALID, "NULL argument");
    int hb, wb;
    int rc = nm_check(frames, bin, window, &hb, &wb);
    if (rc != EPID_OK) return rc;
    EPID_CUDA(cudaSetDevice(ctx->device));
    NmScratch s;
    if ((rc = nm_scratch(ctx, frames->n, hb, wb, true, 0, &s, nullptr)) != EPID_OK) return rc;
    NmPlanes planes = {};
    epid_batch *bc = nullptr, *bm = nullptr;
    if (cleaned) {
        if ((rc = epid_batch_alloc(ctx, EPID_F64, frames->n, hb, wb, &bc)) != EPID_OK) return rc;
        planes.cleaned = (double*)bc->dptr;
    }
    if (masks) {
        if ((rc = epid_batch_alloc(ctx, EPID_U8, 2 * frames->n, hb, wb, &bm)) != EPID_OK) {
            epid_batch_free(bc);
            return rc;
        }
        planes.masks = (uint8_t*)bm->dptr;
    }
    rc = nm_launch(ctx, frames, bin, ufov_erode, cfov_erode, window, threshold, s, hb, wb, planes);
    cudaError_t e = rc == EPID_OK ? cudaMemcpyAsync(results, s.res, frames->n * sizeof(epid_nm_result), cudaMemcpyDeviceToHost, ctx->stream)
                                  : cudaSuccess;
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (rc == EPID_OK && e != cudaSuccess) {
        set_error("nuclear uniformity failed: %s", cudaGetErrorString(e));
        rc = EPID_ERR_CUDA;
    }
    if (rc != EPID_OK) {
        epid_batch_free(bc);
        epid_batch_free(bm);
        return rc;
    }
    if (cleaned) *cleaned = bc;
    if (masks) *masks = bm;
    return EPID_OK;
}

extern "C" int32_t epid_nm_stages(epid_ctx* ctx, const epid_batch* frames, int32_t bin, double ufov_erode, double cfov_erode,
                                  int32_t window, double threshold, struct epid_nm_result* results, uint32_t* filtered, uint32_t* cleaned,
                                  int32_t* edt2, uint8_t* masks) {
    EPID_REQUIRE(ctx && results && filtered && cleaned && edt2 && masks, EPID_ERR_INVALID, "NULL argument");
    int hb, wb;
    int rc = nm_check(frames, bin, window, &hb, &wb);
    if (rc != EPID_OK) return rc;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t plane = (size_t)frames->n * hb * wb;
    const size_t b4 = align256(4 * plane);
    NmScratch s;
    char* extra = nullptr;
    if ((rc = nm_scratch(ctx, frames->n, hb, wb, true, 3 * b4 + align256(2 * plane), &s, &extra)) != EPID_OK) return rc;
    NmPlanes planes = {};
    planes.filtered = (uint32_t*)extra;
    planes.clean_s = (uint32_t*)(extra + b4);
    planes.edt2 = (int32_t*)(extra + 2 * b4);
    planes.masks = (uint8_t*)(extra + 3 * b4);
    EPID_CUDA(cudaMemsetAsync(planes.edt2, 0xff, 4 * plane, ctx->stream));    // -1 where a frame stops before its EDT
    EPID_CUDA(cudaMemsetAsync(planes.masks, 0, 2 * plane, ctx->stream));
    if ((rc = nm_launch(ctx, frames, bin, ufov_erode, cfov_erode, window, threshold, s, hb, wb, planes)) != EPID_OK) return rc;
    EPID_CUDA(cudaMemcpyAsync(results, s.res, frames->n * sizeof(epid_nm_result), cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(filtered, planes.filtered, 4 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(cleaned, planes.clean_s, 4 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(edt2, planes.edt2, 4 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(masks, planes.masks, 2 * plane, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    return EPID_OK;
}

extern "C" int32_t epid_nm_fov(epid_ctx* ctx, const epid_batch* binary, double erode, struct epid_nm_result* results, epid_batch** mask) {
    EPID_REQUIRE(ctx && binary && results && mask, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(binary->dtype == EPID_U8, EPID_ERR_INVALID, "the FOV binary must be uint8 (dtype %d)", binary->dtype);
    EPID_REQUIRE((long long)binary->h * binary->w < (1LL << 30), EPID_ERR_UNSUPPORTED, "frame %d x %d is too large", binary->h, binary->w);
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = binary->n, hb = binary->h, wb = binary->w;
    NmScratch s;
    int rc = nm_scratch(ctx, n, hb, wb, false, align256(2 * (size_t)n * hb * wb), &s, nullptr);
    if (rc != EPID_OK) return rc;
    epid_batch* bm = nullptr;
    if ((rc = epid_batch_alloc(ctx, EPID_U8, 2 * n, hb, wb, &bm)) != EPID_OK) return rc;
    NmPlanes planes = {};
    planes.masks = (uint8_t*)bm->dptr;
    cudaError_t e = cudaSuccess;
    rc = smem_opt_in(ctx, k_nm_frame<uint8_t, false>, s.smem);
    if (rc == EPID_OK) {
        k_nm_frame<uint8_t, false><<<n, NM_THREADS, s.smem, ctx->stream>>>((const uint8_t*)binary->dptr, hb, wb, erode, erode, 1, 0.0,
                                                                           s.use_smem, s.ws, s.res, planes);
        ctx->launches += 1;
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(results, s.res, n * sizeof(epid_nm_result), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            set_error("nuclear FOV failed: %s", cudaGetErrorString(e));
            rc = EPID_ERR_CUDA;
        }
    }
    if (rc != EPID_OK) {
        epid_batch_free(bm);
        return rc;
    }
    *mask = bm;
    return EPID_OK;
}
