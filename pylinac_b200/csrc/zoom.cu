// scipy.ndimage.zoom(order 1 / 3, mode 'constant' / 'nearest', prefilter=True, grid_mode=False) for batches of 2-D frames or 1-D
// profiles (core/image.py:169-220 equate_images; core/profile.py:355-397 as_resampled).
//
//   output shape = round(input shape * zoom); output sample o reads input coordinate o * (n_in - 1) / (n_out - 1)
//   order 3: the B-spline coefficients c solve (c[k-1] + 4 c[k] + c[k+1]) / 6 = s[k] along every axis with mirror boundaries
//            (c[-1] = c[1]); scipy runs the equivalent recursive filter.  Here the tridiagonal system is solved directly (Thomas
//            sweep per line, elimination factors tabulated once): same coefficients to ~1e-16 relative.  mode 'nearest' pads 12
//            edge samples before filtering like scipy's _prepad_for_spline_filter.
//   grid_mode (bit 1 of `mode`, with 'nearest'): output sample o reads (o + 0.5) * n_in / n_out - 0.5 (PhysicalProfileMixin.as_resampled,
//            core/profile.py:951-1013)
//   evaluation: tensor product of the 4 (order 3) or 2 (order 1) B-spline weights at the fractional position, taps outside the
//            array mirrored.
// Validated against scipy.ndimage.zoom on random inputs (tests/test_gpu_primitives.py): max |difference| ~ 1e-13 relative.
#include <cmath>
#include <vector>

#include "common.cuh"

namespace epid {

template <typename T>
__global__ void k_zoom_load(const T* __restrict__ in, int n, int H, int W, int pad_y, int pad_x, double* __restrict__ out) {
    // float64 copy with `pad` edge-replicated samples on either side of the zoomed axes (mode 'nearest')
    const int Hp = H + 2 * pad_y, Wp = W + 2 * pad_x;
    const size_t total = (size_t)n * Hp * Wp;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wp), y = (int)((i / Wp) % Hp), f = (int)(i / ((size_t)Wp * Hp));
        const int sy = min(max(y - pad_y, 0), H - 1), sx = min(max(x - pad_x, 0), W - 1);
        out[i] = (double)in[((size_t)f * H + sy) * W + sx];
    }
}

// Thomas sweep along one axis of every frame: lines = the other axis x frames; cp / im: elimination tables of the axis length
__global__ void k_spline_solve(double* __restrict__ a, int n, int H, int W, int axis, const double* __restrict__ cp, const double* __restrict__ im) {
    const int len = axis == 0 ? H : W, nlines = axis == 0 ? W : H;
    const size_t line = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (line >= (size_t)n * nlines) return;
    const int f = (int)(line / nlines), l = (int)(line % nlines);
    double* p = a + (size_t)f * H * W + (axis == 0 ? l : (size_t)l * W);
    const size_t st = axis == 0 ? W : 1;
    if (len < 2) return;
    // forward: dp[k] = (d[k] - a_k dp[k-1]) / m_k with a_k = 1/6 (2/6 in the last row: mirror)
    double prev = p[0] * im[0];
    p[0] = prev;
    for (int k = 1; k < len; k++) {
        const double ak = k == len - 1 ? 2.0 / 6.0 : 1.0 / 6.0;
        prev = (p[k * st] - ak * prev) * im[k];
        p[k * st] = prev;
    }
    for (int k = len - 2; k >= 0; k--) {
        prev = p[k * st] - cp[k] * prev;
        p[k * st] = prev;
    }
}

__device__ __forceinline__ int mirror_idx(int i, int n) {
    if (n == 1) return 0;
    const int p = 2 * (n - 1);
    i %= p;
    if (i < 0) i += p;
    return i < n ? i : p - i;
}

__global__ void k_zoom_eval(const double* __restrict__ c, int n, int Hp, int Wp, int Ho, int Wo, double zy, double zx, int pad_y, int pad_x,
                            int order, int zoom_y_axis, int grid_mode, double* __restrict__ out) {
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
    if (ox >= Wo || oy >= Ho) return;
    const double* cf = c + (size_t)f * Hp * Wp;
    auto taps = [&](double cc, int* start, double* w) {
        const double fl = floor(cc);
        const double t = cc - fl;
        if (order == 3) {
            const double z = 1.0 - t;
            w[1] = (t * t * (t - 2.0) * 3.0 + 4.0) / 6.0;
            w[2] = (z * z * (z - 2.0) * 3.0 + 4.0) / 6.0;
            w[0] = z * z * z / 6.0;
            w[3] = 1.0 - w[0] - w[1] - w[2];
            *start = (int)fl - 1;
        } else {
            w[0] = 1.0 - t; w[1] = 1.0 - w[0]; w[2] = 0.0; w[3] = 0.0;      // scipy: the last weight is 1 - the others
            *start = (int)fl;
        }
    };
    int sx, sy = 0;
    double wx[4], wy[4] = {1.0, 0.0, 0.0, 0.0};
    // NI_ZoomShift: grid_mode samples pixel CENTRES of a common extent, (o + 0.5) * zoom - 0.5; 'nearest' clamps the (padded) coordinate
    auto coord = [&](int o, double z, int pad, int len) {
        double cc = grid_mode ? ((double)o + 0.5) * z - 0.5 : (double)o * z;
        cc += (double)pad;
        return fmin(fmax(cc, 0.0), (double)(len - 1));
    };
    taps(coord(ox, zx, pad_x, Wp), &sx, wx);
    const int nt = order == 3 ? 4 : 2;
    int nty = 1;
    if (zoom_y_axis) { taps(coord(oy, zy, pad_y, Hp), &sy, wy); nty = nt; } else sy = oy;
    double acc = 0.0;
    for (int j = 0; j < nty; j++) {
        const int yy = zoom_y_axis ? mirror_idx(sy + j, Hp) : sy;
        double row = 0.0;
        for (int i = 0; i < nt; i++) row += wx[i] * cf[(size_t)yy * Wp + mirror_idx(sx + i, Wp)];
        acc += wy[j] * row;
    }
    out[((size_t)f * Ho + oy) * Wo + ox] = acc;
}

static void thomas_tables(int len, std::vector<double>& cp, std::vector<double>& im) {
    cp.assign(len, 0.0);
    im.assign(len, 0.0);
    if (len < 2) return;
    const double b = 4.0 / 6.0;
    // row 0: b x0 + (2/6) x1 (mirror); interior: (1/6, b, 1/6); last row: (2/6) x_{n-2} + b x_{n-1}
    double m = b;
    im[0] = 1.0 / m;
    cp[0] = (2.0 / 6.0) / m;
    for (int k = 1; k < len; k++) {
        const double ak = k == len - 1 ? 2.0 / 6.0 : 1.0 / 6.0;
        m = b - ak * cp[k - 1];
        im[k] = 1.0 / m;
        cp[k] = (1.0 / 6.0) / m;
    }
}

template <typename T>
static int do_zoom_load(epid_ctx* ctx, const epid_batch* in, int pad_y, int pad_x, double* dst) {
    k_zoom_load<T><<<1024, 256, 0, ctx->stream>>>((const T*)in->dptr, in->n, in->h, in->w, pad_y, pad_x, dst);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_zoom(epid_ctx* ctx, const epid_batch* in, double zoom, int32_t order, int32_t mode, epid_batch** out) {
    EPID_REQUIRE(ctx && in && out, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(order == 1 || order == 3, EPID_ERR_UNSUPPORTED, "spline order %d is not supported (1 or 3)", order);
    const int grid_mode = (mode >> 1) & 1;
    mode &= 1;
    EPID_REQUIRE(!grid_mode || mode == 1, EPID_ERR_UNSUPPORTED, "grid_mode zoom is implemented for mode 'nearest' only");
    EPID_REQUIRE(zoom > 0, EPID_ERR_INVALID, "zoom must be positive");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const bool one_d = in->h == 1;                       // profiles: only the sample axis is zoomed
    const int H = in->h, W = in->w;
    const int Ho = one_d ? 1 : (int)nearbyint((double)H * zoom), Wo = (int)nearbyint((double)W * zoom);      // Python round(): half to even
    EPID_REQUIRE(Ho >= 1 && Wo >= 1, EPID_ERR_INVALID, "zoom %g leaves an empty array", zoom);
    const int pad = (mode == 1 && order > 1) ? 12 : 0;   // _prepad_for_spline_filter
    const int pad_y = one_d ? 0 : pad, pad_x = pad;
    const int Hp = H + 2 * pad_y, Wp = W + 2 * pad_x;
    const size_t cbytes = sizeof(double) * (size_t)in->n * Hp * Wp;
    const size_t tbytes = sizeof(double) * 2 * (size_t)(Hp + Wp);
    int rc = ensure_scratch(ctx, cbytes + tbytes + 1024);
    if (rc != EPID_OK) return rc;
    double* coef = (double*)ctx->scratch;
    double* tab = (double*)((char*)ctx->scratch + (cbytes + 255) / 256 * 256);
    rc = epid_batch_alloc(ctx, EPID_F64, in->n, Ho, Wo, out);
    if (rc != EPID_OK) return rc;
    switch (in->dtype) {
        case EPID_U8: rc = do_zoom_load<uint8_t>(ctx, in, pad_y, pad_x, coef); break;
        case EPID_U16: rc = do_zoom_load<uint16_t>(ctx, in, pad_y, pad_x, coef); break;
        case EPID_I16: rc = do_zoom_load<int16_t>(ctx, in, pad_y, pad_x, coef); break;
        case EPID_I32: rc = do_zoom_load<int32_t>(ctx, in, pad_y, pad_x, coef); break;
        case EPID_I64: rc = do_zoom_load<long long>(ctx, in, pad_y, pad_x, coef); break;
        case EPID_F32: rc = do_zoom_load<float>(ctx, in, pad_y, pad_x, coef); break;
        case EPID_F64: rc = do_zoom_load<double>(ctx, in, pad_y, pad_x, coef); break;
        default: set_error("unknown dtype %d", in->dtype); rc = EPID_ERR_INVALID;
    }
    if (rc == EPID_OK && order == 3) {
        std::vector<double> cp, im;
        for (int axis = one_d ? 1 : 0; axis < 2 && rc == EPID_OK; axis++) {      // scipy filters axis 0 first
            const int len = axis == 0 ? Hp : Wp;
            if (len < 2) continue;
            thomas_tables(len, cp, im);
            double* d_cp = tab + (axis == 0 ? 0 : 2 * Hp);
            double* d_im = d_cp + len;
            cudaMemcpyAsync(d_cp, cp.data(), sizeof(double) * len, cudaMemcpyHostToDevice, ctx->stream);
            cudaMemcpyAsync(d_im, im.data(), sizeof(double) * len, cudaMemcpyHostToDevice, ctx->stream);
            cudaStreamSynchronize(ctx->stream);      // the host vectors are reused for the next axis
            const size_t nlines = (size_t)in->n * (axis == 0 ? Wp : Hp);
            k_spline_solve<<<(unsigned)((nlines + 127) / 128), 128, 0, ctx->stream>>>(coef, in->n, Hp, Wp, axis, d_cp, d_im);
            ctx->launches++;
        }
    }
    if (rc == EPID_OK) {
        double zy = Ho > 1 ? (double)(H - 1) / (double)(Ho - 1) : 1.0, zx = Wo > 1 ? (double)(W - 1) / (double)(Wo - 1) : 1.0;
        if (grid_mode) { zy = (double)H / (double)Ho; zx = (double)W / (double)Wo; }
        const dim3 block(32, 8), grid((Wo + 31) / 32, (Ho + 7) / 8, in->n);
        k_zoom_eval<<<grid, block, 0, ctx->stream>>>(coef, in->n, Hp, Wp, Ho, Wo, zy, zx, pad_y, pad_x, order, one_d ? 0 : 1, grid_mode, (double*)(*out)->dptr);
        ctx->launches++;
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (rc == EPID_OK && e != cudaSuccess) { set_error("zoom failed: %s", cudaGetErrorString(e)); rc = EPID_ERR_CUDA; }
    if (rc != EPID_OK) { epid_batch_free(*out); *out = nullptr; }
    return rc;
}

// ------------------------------------------------------------------------------------------------ rotation
// skimage.transform.rotate(image, angle, resize=False, order=1, mode='edge' | 'constant', clip=True, preserve_range=False) as
// BaseImage.rotate calls it (core/image.py:780-783): the image is converted to float first (img_as_float: uint8 / 255, uint16 /
// 65535, floats unchanged), every output pixel (x, y) samples the input bilinearly at R(angle) (x - c, y - c) + c with
// c = (cols / 2 - 0.5, rows / 2 - 0.5), taps outside the frame clamped to the edge ('edge') or read as 0 ('constant').  A bilinear
// sample is a convex combination of four input pixels, so the reference's final clip to the input range is the identity.
// scikit-image is not installed here: restated from its documented algorithm (transform/_warps.py rotate / warp, _warps_cy.pyx
// bilinear_interpolation), validated against scipy.ndimage.affine_transform(order=1) on the same matrix.
namespace epid {

template <typename T>
__global__ void k_rotate(const T* __restrict__ in, int n, int H, int W, double ca, double sa, double cx, double cy, double scale, int mode,
                         double* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
    if (x >= W || y >= H) return;
    const T* __restrict__ src = in + (size_t)f * H * W;
    const double dx = (double)x - cx, dy = (double)y - cy;
    const double c = ca * dx - sa * dy + cx, r = sa * dx + ca * dy + cy;
    const double fr = floor(r), fc = floor(c);
    const long r0 = (long)fr, c0 = (long)fc, r1 = (long)ceil(r), c1 = (long)ceil(c);
    const double dr = r - fr, dc = c - fc;
    auto px = [&](long rr, long cc) -> double {
        if (mode == 0) {
            if (rr < 0 || rr >= H || cc < 0 || cc >= W) return 0.0;
        } else {
            rr = rr < 0 ? 0 : (rr >= H ? H - 1 : rr);
            cc = cc < 0 ? 0 : (cc >= W ? W - 1 : cc);
        }
        return (double)src[rr * W + cc] * scale;
    };
    const double top = (1 - dc) * px(r0, c0) + dc * px(r0, c1);
    const double bot = (1 - dc) * px(r1, c0) + dc * px(r1, c1);
    out[((size_t)f * H + y) * W + x] = (1 - dr) * top + dr * bot;
}

template <typename T>
static void launch_rotate(epid_ctx* ctx, const epid_batch* in, double ca, double sa, double scale, int mode, double* out) {
    const dim3 block(32, 8), grid((in->w + 31) / 32, (in->h + 7) / 8, in->n);
    k_rotate<T><<<grid, block, 0, ctx->stream>>>((const T*)in->dptr, in->n, in->h, in->w, ca, sa, in->w / 2.0 - 0.5, in->h / 2.0 - 0.5, scale,
                                                  mode, out);
    ctx->launches++;
}

}  // namespace epid

extern "C" int32_t epid_rotate(epid_ctx* ctx, const epid_batch* in, double angle_deg, int32_t mode, epid_batch** out) {
    EPID_REQUIRE(ctx && in && out, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(mode == 0 || mode == 1, EPID_ERR_UNSUPPORTED, "rotate mode must be 0 (constant) or 1 (edge)");
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = epid_batch_alloc(ctx, EPID_F64, in->n, in->h, in->w, out);
    if (rc != EPID_OK) return rc;
    const double a = angle_deg * 3.14159265358979323846 / 180.0;
    const double ca = cos(a), sa = sin(a);
    double* dst = (double*)(*out)->dptr;
    switch (in->dtype) {
        case EPID_U8: launch_rotate<uint8_t>(ctx, in, ca, sa, 1.0 / 255.0, mode, dst); break;
        case EPID_U16: launch_rotate<uint16_t>(ctx, in, ca, sa, 1.0 / 65535.0, mode, dst); break;
        case EPID_F32: launch_rotate<float>(ctx, in, ca, sa, 1.0, mode, dst); break;
        case EPID_F64: launch_rotate<double>(ctx, in, ca, sa, 1.0, mode, dst); break;
        default: set_error("rotate: dtype %d is not supported (uint8, uint16, float32, float64)", in->dtype); rc = EPID_ERR_UNSUPPORTED;
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (rc == EPID_OK && e != cudaSuccess) { set_error("rotate failed: %s", cudaGetErrorString(e)); rc = EPID_ERR_CUDA; }
    if (rc != EPID_OK) { epid_batch_free(*out); *out = nullptr; }
    return rc;
}
