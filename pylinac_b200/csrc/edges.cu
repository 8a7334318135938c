// Edge and line operators of JawOrthogonality.analyze (contrib/orthogonality.py:29-50): skimage.feature.canny,
// skimage.transform.hough_line and the device half of hough_line_peaks, restated from the published algorithms (scikit-image is not
// available in the build container and the reference holds no vectors for this path: PARITY UNPINNED, see oracle/edges_oracle.py).
//
//   epid_canny        float64 frames -> uint8 edge maps.  k_canny_gauss_v / k_canny_gauss_h: scipy.ndimage.gaussian_filter(sigma,
//                     mode='constant', truncate=4) as two correlate1d passes in scipy's symmetric summation order, divided by the
//                     same filter of an all-ones mask (+ eps): skimage's bleed-over correction; k_canny_grad: ndimage.sobel along both
//                     axes (mode 'reflect', scipy's anti-/symmetric summation order) + magnitude; k_canny_nms: bilinear non-maximum
//                     suppression along the gradient; hysteresis = 8-connected components of the low mask (k_ccl_union,
//                     ccl.cuh) that contain a pixel >= the high threshold.
//   epid_hough_line   every edge pixel votes for round(x cos t + y sin t) + offset at every angle (uint32 atomics on an L2-resident
//                     accumulator): accumulator [2 * offset + 1][ntheta] as an int32 batch.
//   epid_hough_candidates   _prominent_peaks up to its thresholded local maxima: separable maximum filter (mode 'constant'), pixels
//                     equal to their local maximum and above the threshold, compacted to a list; the filtered accumulator stays on
//                     the device for epid_gather_i32 (the component / suppression bookkeeping of the few surviving points is scalar
//                     work in the binding).
#include <algorithm>
#include <cmath>
#include <vector>

#include "ccl.cuh"
#include "common.cuh"

namespace epid {

constexpr int ED_THREADS = 256;
constexpr int ED_MAXR = 64;      // gaussian radius limit (sigma <= 15)

struct GaussW { int r; double w[ED_MAXR + 1]; };      // w[0..r]: weights of offsets -r .. 0 (symmetric kernel)

// correlate1d, symmetric case, mode 'constant' (cval 0): tmp = in[l] w[r]; for ii = -r .. -1: tmp += (in[l + ii] + in[l - ii]) w[ii + r]
__global__ void k_canny_gauss_v(const double* __restrict__ in, double* __restrict__ out, int H, int W, GaussW g) {
    const int f = blockIdx.z;
    const size_t o = (size_t)f * H * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    auto at = [&](int yy) { return (yy >= 0 && yy < H) ? in[o + (size_t)yy * W + x] : 0.0; };
    double t = at(y) * g.w[g.r];
    for (int ii = -g.r; ii < 0; ii++) t += (at(y + ii) + at(y - ii)) * g.w[ii + g.r];
    out[o + (size_t)y * W + x] = t;
}

__global__ void k_canny_gauss_h(const double* __restrict__ in, double* __restrict__ out, int H, int W, GaussW g) {
    const int f = blockIdx.z;
    const size_t o = (size_t)f * H * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const double* row = in + o + (size_t)y * W;
    auto at = [&](int xx) { return (xx >= 0 && xx < W) ? row[xx] : 0.0; };
    double t = at(x) * g.w[g.r];
    for (int ii = -g.r; ii < 0; ii++) t += (at(x + ii) + at(x - ii)) * g.w[ii + g.r];
    // the same two passes over an all-ones image: first along y (depends on y only), then along x
    auto one_y = [&](int yy) { return (yy >= 0 && yy < H) ? 1.0 : 0.0; };
    double by = one_y(y) * g.w[g.r];
    for (int ii = -g.r; ii < 0; ii++) by += (one_y(y + ii) + one_y(y - ii)) * g.w[ii + g.r];
    auto b_at = [&](int xx) { return (xx >= 0 && xx < W) ? by : 0.0; };
    double bl = b_at(x) * g.w[g.r];
    for (int ii = -g.r; ii < 0; ii++) bl += (b_at(x + ii) + b_at(x - ii)) * g.w[ii + g.r];
    out[o + (size_t)y * W + x] = t / (bl + 2.220446049250313e-16);
}

__device__ __forceinline__ int refl(int i, int n) { return i < 0 ? -i - 1 : (i >= n ? 2 * n - 1 - i : i); }

// ndimage.sobel(s, axis=1) -> jsobel, ndimage.sobel(s, axis=0) -> isobel; magnitude = sqrt(i * i + j * j)
__global__ void k_canny_grad(const double* __restrict__ s, double* __restrict__ isob, double* __restrict__ jsob, double* __restrict__ mag, int H, int W) {
    const int f = blockIdx.z;
    const size_t o = (size_t)f * H * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const int xm = refl(x - 1, W), xp = refl(x + 1, W), ym = refl(y - 1, H), yp = refl(y + 1, H);
    auto S = [&](int yy, int xx) { return s[o + (size_t)yy * W + xx]; };
    // derivative along x of a row: in[x] * 0 + (in[x-1] - in[x+1]) * (-1)   (correlate1d, antisymmetric weights [-1, 0, 1])
    auto dx = [&](int yy) { return S(yy, x) * 0.0 + (S(yy, xm) - S(yy, xp)) * -1.0; };
    auto dy = [&](int xx) { return S(y, xx) * 0.0 + (S(ym, xx) - S(yp, xx)) * -1.0; };
    // smoothing [1, 2, 1] along the other axis: in[l] * 2 + (in[l-1] + in[l+1]) * 1
    const double j = dx(y) * 2.0 + (dx(ym) + dx(yp)) * 1.0;
    const double i = dy(x) * 2.0 + (dy(xm) + dy(xp)) * 1.0;
    double m = i * i;
    m += j * j;
    const size_t k = o + (size_t)y * W + x;
    isob[k] = i; jsob[k] = j; mag[k] = sqrt(m);
}

__global__ void k_canny_nms(const double* __restrict__ isob, const double* __restrict__ jsob, const double* __restrict__ mag, double* __restrict__ out,
                            int H, int W, double low) {
    const int f = blockIdx.z;
    const size_t o = (size_t)f * H * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;      // y: row ("x" of the cython loop), x: column ("y")
    if (x >= W) return;
    const size_t k = o + (size_t)y * W + x;
    double res = 0.0;
    if (y >= 1 && y < H - 1 && x >= 1 && x < W - 1) {      // eroded mask (outer frame excluded) and the loop bounds coincide
        const double m = mag[k];
        if (m >= low) {
            const double iv = isob[k], jv = jsob[k];
            const bool is_down = iv <= 0, is_up = iv >= 0, is_left = jv <= 0, is_right = jv >= 0;
            const bool cond1 = (is_up && is_right) || (is_down && is_left), cond2 = (is_down && is_right) || (is_up && is_left);
            if (cond1 || cond2) {
                const double ai = fabs(iv), aj = fabs(jv);
                const bool g1 = ai > aj;
                const double w = g1 ? aj / ai : ai / aj;
                auto M = [&](int dy, int dx) { return mag[o + (size_t)(y + dy) * W + (x + dx)]; };
                double n11, n12, n21, n22;
                if (cond1) {
                    if (g1) { n11 = M(1, 0); n12 = M(1, 1); n21 = M(-1, 0); n22 = M(-1, -1); }
                    else { n11 = M(0, 1); n12 = M(1, 1); n21 = M(0, -1); n22 = M(-1, -1); }
                } else {
                    if (g1) { n11 = M(-1, 0); n12 = M(-1, 1); n21 = M(1, 0); n22 = M(1, -1); }
                    else { n11 = M(0, 1); n12 = M(-1, 1); n21 = M(0, -1); n22 = M(1, -1); }
                }
                const bool c_plus = (n12 * w + n11 * (1.0 - w)) <= m;
                if (c_plus && (n22 * w + n21 * (1.0 - w)) <= m) res = m;
            }
        }
    }
    out[k] = res;
}

__global__ void k_hyst_init(const double* __restrict__ lowm, int* __restrict__ parent, int* __restrict__ good, int HW) {
    const int f = blockIdx.y;
    const size_t o = (size_t)f * HW;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        parent[o + i] = lowm[o + i] > 0 ? i : -1;
        good[o + i] = 0;
    }
}

__global__ void k_hyst_mark(const double* __restrict__ lowm, int* __restrict__ parent, int* __restrict__ good, int HW, double high) {
    const int f = blockIdx.y;
    const size_t o = (size_t)f * HW;
    int* par = parent + o;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        if (par[i] < 0) continue;
        const int r = ccl_root(par, i);
        if (r != i) par[i] = r;
        if (lowm[o + i] >= high) good[o + r] = 1;
    }
}

__global__ void k_hyst_out(const int* __restrict__ parent, const int* __restrict__ good, uint8_t* __restrict__ out, int HW) {
    const int f = blockIdx.y;
    const size_t o = (size_t)f * HW;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        int r = parent[o + i];
        if (r >= 0) { const int p = parent[o + r]; if (p != r) r = p; }
        out[o + i] = (r >= 0 && good[o + r]) ? 1 : 0;
    }
}

// ------------------------------------------------------------------------------------------------ Hough
__global__ void k_hough_vote(const uint8_t* __restrict__ edges, int H, int W, int ntheta, const double* __restrict__ ct, const double* __restrict__ st,
                             int offset, unsigned int* __restrict__ accum) {
    // one CTA per image row: its edge pixels are collected first, then every thread walks angles for every collected pixel
    const int y = blockIdx.x;
    __shared__ int s_x[2048];
    __shared__ int s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += blockDim.x)
        if (edges[(size_t)y * W + x]) { const int k = atomicAdd(&s_n, 1); if (k < 2048) s_x[k] = x; }
    __syncthreads();
    const int n = min(s_n, 2048);
    for (int p = 0; p < n; p++) {
        const double xd = (double)s_x[p], yd = (double)y;
        for (int j = threadIdx.x; j < ntheta; j += blockDim.x) {
            const double r = ct[j] * xd + st[j] * yd;
            const long long idx = (long long)(r > 0.0 ? r + 0.5 : r - 0.5) + offset;      // skimage's round(): truncation of r +- 0.5
            atomicAdd(&accum[(size_t)idx * ntheta + j], 1u);
        }
    }
}

// maximum_filter1d(size = 2 d + 1, mode='constant', cval=0) along rows (axis 0) / columns (axis 1) of a [R][C] int32 image
__global__ void k_maxfilt_axis0(const int* __restrict__ in, int* __restrict__ out, int R, int C, int d) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= C) return;
    int m = 0;      // cval 0 takes part whenever the window leaves the array; counts are >= 0 anyway
    for (int k = max(r - d, 0); k <= min(r + d, R - 1); k++) m = max(m, in[(size_t)k * C + c]);
    out[(size_t)r * C + c] = m;
}
__global__ void k_maxfilt_axis1(const int* __restrict__ in, int* __restrict__ out, int R, int C, int d) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= C) return;
    int m = 0;
    for (int k = max(c - d, 0); k <= min(c + d, C - 1); k++) m = max(m, in[(size_t)r * C + k]);
    out[(size_t)r * C + c] = m;
}

__global__ void k_max_all(const int* __restrict__ in, size_t n, int* __restrict__ out) {
    int m = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) m = max(m, in[i]);
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void k_peak_candidates(const int* __restrict__ img, const int* __restrict__ img_max, int R, int C, double threshold, const int* __restrict__ gmax,
                                  int cap, int* __restrict__ cand, int* __restrict__ count) {
    const double thr = threshold >= 0 ? threshold : 0.5 * (double)*gmax;
    const size_t n = (size_t)R * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int v = img[i];
        if (v == img_max[i] && (double)v > thr) {
            const int k = atomicAdd(count, 1);
            if (k < cap) { cand[3 * k] = (int)(i / C); cand[3 * k + 1] = (int)(i % C); cand[3 * k + 2] = v; }
        }
    }
}

__global__ void k_gather_i32(const int* __restrict__ img, int R, int C, const int* __restrict__ yx, int n, int* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int y = yx[2 * i], x = yx[2 * i + 1];
    out[i] = (y >= 0 && y < R && x >= 0 && x < C) ? img[(size_t)y * C + x] : 0;
}

}  // namespace epid

using namespace epid;

static int no_device() {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device"); return 1; }
    return 0;
}

extern "C" int32_t epid_canny(epid_ctx* ctx, const epid_batch* in, const double* weights, int32_t radius, double low_threshold,
                              double high_threshold, epid_batch** out) {
    EPID_REQUIRE(ctx && in && out && weights, EPID_ERR_INVALID, "NULL argument");
    if (no_device()) return EPID_ERR_NO_DEVICE;
    EPID_REQUIRE(in->dtype == EPID_F64, EPID_ERR_UNSUPPORTED, "epid_canny takes float64 frames (the stretched image)");
    EPID_REQUIRE(radius >= 0 && radius <= ED_MAXR, EPID_ERR_INVALID, "gaussian radius out of range");
    EPID_REQUIRE(in->h >= 3 && in->w >= 3 && (size_t)in->h * in->w < 0x7fffffff, EPID_ERR_INVALID, "frame shape unsupported");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = in->n, H = in->h, W = in->w;
    const size_t per = (size_t)H * W, total = per * n;
    // weights: scipy's _gaussian_kernel1d(sigma, 0, radius) (2 * radius + 1 values) computed by the binding with the same numpy
    // expression scipy evaluates; the kernel is symmetric, the left half + centre are used like scipy's symmetric correlate1d does
    GaussW g;
    g.r = radius;
    for (int k = 0; k <= radius; k++) g.w[k] = weights[k];
    auto rup = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t bd = rup(sizeof(double) * total), bi = rup(sizeof(int) * total);
    int rc = ensure_scratch(ctx, 5 * bd + 2 * bi + 1024);
    if (rc != EPID_OK) return rc;
    char* q = (char*)ctx->scratch;
    double* d_tmp = (double*)q; q += bd;
    double* d_sm = (double*)q; q += bd;
    double* d_i = (double*)q; q += bd;
    double* d_j = (double*)q; q += bd;
    double* d_mag = (double*)q; q += bd;
    int* d_par = (int*)q; q += bi;
    int* d_good = (int*)q;
    rc = epid_batch_alloc(ctx, EPID_U8, n, H, W, out);
    if (rc != EPID_OK) return rc;
    const dim3 grid((W + ED_THREADS - 1) / ED_THREADS, H, n);
    cudaStream_t st = ctx->stream;
    k_canny_gauss_v<<<grid, ED_THREADS, 0, st>>>((const double*)in->dptr, d_tmp, H, W, g);
    k_canny_gauss_h<<<grid, ED_THREADS, 0, st>>>(d_tmp, d_sm, H, W, g);
    k_canny_grad<<<grid, ED_THREADS, 0, st>>>(d_sm, d_i, d_j, d_mag, H, W);
    k_canny_nms<<<grid, ED_THREADS, 0, st>>>(d_i, d_j, d_mag, d_tmp, H, W, low_threshold);      // d_tmp = low_masked
    const dim3 g2(ctx->sm_count * 2, n);
    k_hyst_init<<<g2, 256, 0, st>>>(d_tmp, d_par, d_good, (int)per);
    k_ccl_union<<<g2, 256, 0, st>>>(H, W, 1, d_par);
    k_hyst_mark<<<g2, 256, 0, st>>>(d_tmp, d_par, d_good, (int)per, high_threshold);
    k_hyst_out<<<g2, 256, 0, st>>>(d_par, d_good, (uint8_t*)(*out)->dptr, (int)per);
    ctx->launches += 8;
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaStreamSynchronize(st));
    return EPID_OK;
}

extern "C" int32_t epid_hough_line(epid_ctx* ctx, const epid_batch* edges, int32_t ntheta, const double* theta, epid_batch** accum, int32_t* offset_out) {
    EPID_REQUIRE(ctx && edges && theta && accum && offset_out && ntheta > 0, EPID_ERR_INVALID, "bad argument");
    if (no_device()) return EPID_ERR_NO_DEVICE;
    EPID_REQUIRE(edges->dtype == EPID_U8 && edges->n == 1, EPID_ERR_UNSUPPORTED, "epid_hough_line takes one uint8 edge map");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int H = edges->h, W = edges->w;
    const int offset = (int)ceil(sqrt((double)H * H + (double)W * W));
    const int R = 2 * offset + 1;
    std::vector<double> ct(ntheta), sn(ntheta);
    for (int j = 0; j < ntheta; j++) { ct[j] = cos(theta[j]); sn[j] = sin(theta[j]); }      // libm on the host like numpy
    int rc = ensure_scratch(ctx, 2 * sizeof(double) * ntheta + 512);
    if (rc != EPID_OK) return rc;
    double* d_ct = (double*)ctx->scratch;
    double* d_st = d_ct + ntheta;
    rc = epid_batch_alloc(ctx, EPID_I32, 1, R, ntheta, accum);
    if (rc != EPID_OK) return rc;
    cudaStream_t st = ctx->stream;
    EPID_CUDA(cudaMemcpyAsync(d_ct, ct.data(), sizeof(double) * ntheta, cudaMemcpyHostToDevice, st));
    EPID_CUDA(cudaMemcpyAsync(d_st, sn.data(), sizeof(double) * ntheta, cudaMemcpyHostToDevice, st));
    EPID_CUDA(cudaMemsetAsync((*accum)->dptr, 0, sizeof(int) * (size_t)R * ntheta, st));
    k_hough_vote<<<H, 256, 0, st>>>((const uint8_t*)edges->dptr, H, W, ntheta, d_ct, d_st, offset, (unsigned int*)(*accum)->dptr);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaStreamSynchronize(st));
    *offset_out = offset;
    return EPID_OK;
}

extern "C" int32_t epid_hough_candidates(epid_ctx* ctx, const epid_batch* accum, int32_t min_xdistance, int32_t min_ydistance, double threshold,
                                         int32_t cap, int32_t* cand_yxv, int32_t* count, int32_t* global_max, epid_batch** filtered) {
    EPID_REQUIRE(ctx && accum && cand_yxv && count && global_max && filtered && cap > 0, EPID_ERR_INVALID, "bad argument");
    if (no_device()) return EPID_ERR_NO_DEVICE;
    EPID_REQUIRE(accum->dtype == EPID_I32 && accum->n == 1, EPID_ERR_UNSUPPORTED, "one int32 accumulator expected");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int R = accum->h, C = accum->w;
    const size_t n = (size_t)R * C;
    auto rup = [](size_t b) { return (b + 255) / 256 * 256; };
    int rc = ensure_scratch(ctx, rup(sizeof(int) * n) + rup(sizeof(int) * 3 * (size_t)cap) + 1024);
    if (rc != EPID_OK) return rc;
    char* q = (char*)ctx->scratch;
    int* d_tmp = (int*)q; q += rup(sizeof(int) * n);
    int* d_cand = (int*)q; q += rup(sizeof(int) * 3 * (size_t)cap);
    int* d_cnt = (int*)q;      // [0] count, [1] global max
    rc = epid_batch_alloc(ctx, EPID_I32, 1, R, C, filtered);
    if (rc != EPID_OK) return rc;
    cudaStream_t st = ctx->stream;
    EPID_CUDA(cudaMemsetAsync(d_cnt, 0, 2 * sizeof(int), st));
    const dim3 grid((C + 255) / 256, R);
    k_maxfilt_axis0<<<grid, 256, 0, st>>>((const int*)accum->dptr, d_tmp, R, C, min_ydistance);
    k_maxfilt_axis1<<<grid, 256, 0, st>>>(d_tmp, (int*)(*filtered)->dptr, R, C, min_xdistance);
    k_max_all<<<ctx->sm_count * 2, 256, 0, st>>>((const int*)accum->dptr, n, d_cnt + 1);
    k_peak_candidates<<<ctx->sm_count * 2, 256, 0, st>>>((const int*)accum->dptr, (const int*)(*filtered)->dptr, R, C, threshold, d_cnt + 1, cap, d_cand, d_cnt);
    ctx->launches += 4;
    EPID_CUDA(cudaGetLastError());
    int hc[2] = {0, 0};
    EPID_CUDA(cudaMemcpyAsync(hc, d_cnt, sizeof(hc), cudaMemcpyDeviceToHost, st));
    EPID_CUDA(cudaStreamSynchronize(st));
    *global_max = hc[1];
    EPID_REQUIRE(hc[0] <= cap, EPID_ERR_NOMEM, "%d peak candidates exceed the capacity %d", hc[0], cap);
    *count = hc[0];
    if (hc[0] > 0) {
        EPID_CUDA(cudaMemcpyAsync(cand_yxv, d_cand, sizeof(int) * 3 * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
        EPID_CUDA(cudaStreamSynchronize(st));
    }
    return EPID_OK;
}

extern "C" int32_t epid_gather_i32(epid_ctx* ctx, const epid_batch* img, int32_t npts, const int32_t* yx, int32_t* values) {
    EPID_REQUIRE(ctx && img && yx && values && npts >= 0, EPID_ERR_INVALID, "bad argument");
    if (no_device()) return EPID_ERR_NO_DEVICE;
    EPID_REQUIRE(img->dtype == EPID_I32 && img->n == 1, EPID_ERR_UNSUPPORTED, "one int32 image expected");
    if (npts == 0) return EPID_OK;
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = ensure_scratch(ctx, sizeof(int) * 3 * (size_t)npts + 512);
    if (rc != EPID_OK) return rc;
    int* d_yx = (int*)ctx->scratch;
    int* d_out = d_yx + 2 * (size_t)npts;
    cudaStream_t st = ctx->stream;
    EPID_CUDA(cudaMemcpyAsync(d_yx, yx, sizeof(int) * 2 * (size_t)npts, cudaMemcpyHostToDevice, st));
    k_gather_i32<<<(npts + 127) / 128, 128, 0, st>>>((const int*)img->dptr, img->h, img->w, d_yx, npts, d_out);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaMemcpyAsync(values, d_out, sizeof(int) * (size_t)npts, cudaMemcpyDeviceToHost, st));
    EPID_CUDA(cudaStreamSynchronize(st));
    return EPID_OK;
}
