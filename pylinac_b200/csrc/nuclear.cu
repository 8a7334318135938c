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
#include "nuclear_reduce.cuh"

#include <climits>
#include <cmath>

namespace epid {
namespace {

using namespace nm;

constexpr int NM_BIN_THREADS = 256;
constexpr int NM_BIN_COLS = 2048;      // raw columns per pass of k_nm_bin (a multiple of every supported bin)
constexpr int NM_THREADS = 512;
constexpr int NM_MAX_BIN = 64;         // 16 * 65535 * 64^2 < 2^32: S stays a uint32
constexpr int NM_BIG = 1 << 20;        // column distance of a pixel with no background above / below it

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

    // ---- 4-connected labelling: roots are the smallest index of their component (skimage's raster label order)
    for (int p = tid; p < N; p += nt) {
        if (P[p] < 0) continue;
        const int i = p / wb, j = p - i * wb;
        if (j > 0 && P[p - 1] >= 0) gl_union(P, p, p - 1);
        if (i > 0 && P[p - wb] >= 0) gl_union(P, p, p - wb);
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
    // largest area; on ties the lowest label, i.e. the smallest root index
    unsigned long long key = 0;
    for (int p = tid; p < N; p += nt) {
        if (P[p] != p) continue;
        const unsigned long long k = ((unsigned long long)A[p] << 32) | (0xffffffffu - (uint32_t)p);
        key = k > key ? k : key;
    }
    key = block_reduce(key, OpMax(), red);
    if (key == 0) {               // no component: get_fov's max() over no regions raises
        if (tid == 0) {
            r.status = EPID_NM_NO_COMPONENT;
            res[f] = r;
        }
        return;
    }
    const int root = (int)(0xffffffffu - (uint32_t)key);
    long long rmin = LLONG_MAX, rmax = -1, cmin = LLONG_MAX, cmax = -1;
    for (int p = tid; p < N; p += nt) {
        if (P[p] != root) continue;
        const int i = p / wb, j = p - i * wb;
        rmin = min(rmin, (long long)i);
        rmax = max(rmax, (long long)i);
        cmin = min(cmin, (long long)j);
        cmax = max(cmax, (long long)j);
    }
    rmin = block_reduce(rmin, OpMin(), red);
    rmax = block_reduce(rmax, OpMax(), red);
    cmin = block_reduce(cmin, OpMin(), red);
    cmax = block_reduce(cmax, OpMax(), red);
    const int longest = (int)max(rmax - rmin + 1, cmax - cmin + 1);
    // int(round((1 - size) * longest)): Python rounds halves to even, as rint does
    const int eu = (int)rint(ufov_erode * (double)longest), ec = (int)rint(cfov_erode * (double)longest);
    r.longest = longest;
    r.erosion[0] = eu;
    r.erosion[1] = ec;

    // ---- exact squared EDT of the whole binary frame: column distances, then the row-wise minimum of dk^2 + g^2
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
        if (out.edt2) out.edt2[fo + p] = P[p];
    }
    __syncthreads();

    // ---- FOV masks: distance > erosion / 2  <=>  4 d^2 > erosion^2 (every pixel when the erosion is negative)
    const long long e2[2] = {(long long)eu * eu, (long long)ec * ec};
    const bool all[2] = {eu < 0, ec < 0};
    auto in_fov = [&](int p, int k) { return all[k] || 4LL * P[p] > e2[k]; };
    unsigned long long mxk[2] = {0, 0}, mnk[2] = {~0ull, ~0ull}, nfov[2] = {0, 0};
    for (int p = tid; p < N; p += nt) {
        for (int k = 0; k < 2; k++) {
            const bool m = in_fov(p, k);
            if (out.masks) out.masks[(2 * (size_t)f + k) * N + p] = m;
            if (!m || S[p] == 0) continue;
            const unsigned long long hi = (unsigned long long)S[p] << 32;
            mxk[k] = max(mxk[k], hi | (0xffffffffu - (uint32_t)p));   // max value, first index
            mnk[k] = min(mnk[k], hi | (uint32_t)p);                    // min value, first index
            nfov[k]++;
        }
    }
    for (int k = 0; k < 2; k++) {
        mxk[k] = block_reduce(mxk[k], OpMax(), red);
        mnk[k] = block_reduce(mnk[k], OpMin(), red);
        nfov[k] = block_reduce(nfov[k], OpSum(), red);
        r.n_fov[k] = (int)nfov[k];
        if (nfov[k]) {
            const unsigned long long smx = mxk[k] >> 32, smn = mnk[k] >> 32;
            r.max_index[k] = (int)(0xffffffffu - (uint32_t)mxk[k]);
            r.min_index[k] = (int)(uint32_t)mnk[k];
            r.iu[k] = (double)(smx - smn) / (double)(smx + smn) * 100.0;   // michelson(S / 16) * 100: the 1/16 cancels exactly
        }
    }

    // ---- differential uniformity: windows of `win` pixels along axis 0 (a = 0) and axis 1 (a = 1) over the non-zero FOV pixels; a
    // window counts when it holds at least one.  Per (FOV, axis): the max of the x100 values and its first (i, j) in row-major order.
    for (int k = 0; k < 2; k++) {
        for (int a = 0; a < 2; a++) {
            const int ni = a == 0 ? hb - win + 1 : hb, nj = a == 0 ? wb : wb - win + 1;
            const int step = a == 0 ? wb : 1;
            const long long npos = ni > 0 && nj > 0 ? (long long)ni * nj : 0;
            unsigned long long vbest = 0, cnt = 0;
            for (long long q = tid; q < npos; q += nt) {
                const int i = (int)(q / nj), j = (int)(q - (long long)i * nj);
                uint32_t mx = 0, mn = UINT_MAX;
                for (int t = 0, p = i * wb + j; t < win; t++, p += step) {
                    if (!in_fov(p, k) || S[p] == 0) continue;
                    mx = max(mx, S[p]);
                    mn = min(mn, S[p]);
                }
                if (mx == 0) continue;
                const double v = (double)(mx - mn) / (double)((unsigned long long)mx + mn) * 100.0;
                vbest = max(vbest, (unsigned long long)__double_as_longlong(v));   // v >= 0: the bits order like the values
                cnt++;
            }
            vbest = block_reduce(vbest, OpMax(), red);
            cnt = block_reduce(cnt, OpSum(), red);
            unsigned long long pos = ~0ull;
            for (long long q = tid; q < npos && cnt; q += nt) {
                const int i = (int)(q / nj), j = (int)(q - (long long)i * nj);
                uint32_t mx = 0, mn = UINT_MAX;
                for (int t = 0, p = i * wb + j; t < win; t++, p += step) {
                    if (!in_fov(p, k) || S[p] == 0) continue;
                    mx = max(mx, S[p]);
                    mn = min(mn, S[p]);
                }
                if (mx == 0) continue;
                const double v = (double)(mx - mn) / (double)((unsigned long long)mx + mn) * 100.0;
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
