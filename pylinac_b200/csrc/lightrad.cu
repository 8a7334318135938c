// Light / radiation field coincidence phantoms on device-resident frames (epid_lightrad_analyze).
//
// Reference path reproduced (pylinac v3.46.0):
//   ImagePhantomBase.__init__ ground / normalize                                 planar_imaging.py:226-231
//   StandardImagingFC2.analyze / _find_field_info / _find_overall_bb_centroid /
//     _detect_bb_centers / _determine_bb_set / _is_bb_near_edge                   planar_imaging.py:1282-1305, 1405-1468, 1614-1623
//   IMTLRad / DoselabRLf / IsoAlign / SNCFSQA BB sets                            planar_imaging.py:1626-1727
//   QuasarLightRadScaling._determine_bb_set / _detect_scaling_centers            contrib/quasar.py:27-66
//   BaseImage.check_inversion / filter / invert                                   core/image.py:695-757, 868-897
//   FWXMProfilePhysical(ground=True, normalization=BEAM_CENTER)                   core/profile.py:195-345, 578-611, 742-790, 1016-1047
//   skimage.exposure.equalize_adapthist (restated, UNPINNED: tests/golden/clahe_restated.py)
//
// Exactness (DESIGN 2.1): ground / normalize / invert are a monotone map of the uint16 frame, so the strip sums, the inversion test
// and both 3 x 3 medians are integer work; the once-filtered image is I = (T(median) - mn) / D.  CLAHE quantises that image to 14 bits,
// interpolates integer tile maps in float32 and casts the result back to uint16 before its final rescale to [0, 1]: its output is again
// an affine map (u - umin) / (umax - umin) of integers, and so is the median of it.  Every BB window therefore runs the integer path
// of the windowed locator (k_wl_bb, wl.cu) unchanged.
//
// Stages, one launch sequence per chunk of frames, no host round trip:
//   k_lr_init         per-frame accumulators
//   k_lr_front        one read of the raw frame: min / max / sum, the four 20-pixel corner boxes, the row sums of the vertical strip
//                     and the column sums of the horizontal strip
//   k_lr_profile      CTA per (frame, axis): inversion decision, strip means through the pixel map, FWXM edges, centre, width
//   k_lr_plan         per frame: BB set (mismatch check), near-edge decisions, the value map of the first median
//   median 3 x 3      (filters.cu) of the whole mapped frame
//   k_lr_fminmax      near-edge frames: range of the filtered frame (the 14-bit rescale of equalize_adapthist)
//   k_lr_clahe_maps   warp per contextual region: 256-bin histogram in shared memory, clip + redistribution, cumulative map
//   k_lr_clahe_apply  thread per pixel: bilinear interpolation of the four neighbouring maps, range of the result
//   median 3 x 3      of the equalised frames (near-edge frames only)
//   k_lr_items        one locator item per BB (+ the Quasar scaling search): source frame, pixel map, window
//   k_wl_bb           (wl.cu, launch_disk_items) the windowed disk locator per item
//   k_lr_finalize     per frame: points into the result row, exceptions in the reference's order
// epid_lightrad_stages runs the same sequence and also copies the three planes and the per-frame accumulators back, for the tests.
#include <cmath>
#include <vector>

#include "common.cuh"
#include "filters.cuh"
#include "profile1d.cuh"
#include "stats.cuh"
#include "wl.cuh"

namespace epid {

constexpr int LR_THREADS = 256;
constexpr int LR_PARTS = 16;           // CTAs per frame in the streaming passes
constexpr int LR_NGRAY = 1 << 14;      // NR_OF_GRAY of equalize_adapthist
constexpr int LR_NBINS = 256;
constexpr int LR_BIN = 1 + LR_NGRAY / LR_NBINS;

struct LrFrame {
    unsigned int mn, mx;               // raw range
    unsigned long long sum, corner;    // raw frame sum, raw sum of the four corner boxes
    int checked;                       // check_inversion fired
    int inv;                           // final inversion (check_inversion xor the invert argument)
    int status;
    int near_any;
    int large;
    int near_mask;
    double cx, cy, wx, wy;             // field centre (pixels), widths (mm)
    unsigned int fmn, fmx;             // range of the once-filtered mapped frame (near-edge frames)
    unsigned int umin, umax;           // range of the equalised frame
};

struct LrConst {
    epid_lr_params p;
    int H, W;
    int sx0, sx1, sy0, sy1;            // strip bounds: columns of the vertical strip, rows of the horizontal strip
    int k;                             // CLAHE kernel edge
    int nth, ntw;                      // contextual regions (histogram tiles) per column / row
    int clim;                          // clip limit in counts
    double map_scale;                  // (2**14 - 1) / (k * k)
    int nitems;                        // items per frame
};

__global__ void k_lr_init(LrFrame* fr, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    LrFrame f;
    memset(&f, 0, sizeof(f));
    f.mn = 0xffffffffu;
    f.fmn = 0xffffffffu;
    f.umin = 0xffffffffu;
    fr[i] = f;
}

// ------------------------------------------------------------------------------------------------ front: one read of the raw frame
__global__ void __launch_bounds__(LR_THREADS)
k_lr_front(const LrConst* __restrict__ cc, const uint16_t* __restrict__ base, LrFrame* fr, unsigned long long* __restrict__ ysum,
           unsigned long long* __restrict__ xsum) {
    __shared__ unsigned int s_mn[LR_THREADS / 32], s_mx[LR_THREADS / 32];
    __shared__ unsigned long long s_sum[LR_THREADS / 32], s_cor[LR_THREADS / 32];
    const LrConst& c = *cc;
    const int H = c.H, W = c.W, fi = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint16_t* f = base + (size_t)fi * H * W;
    unsigned long long* ys = ysum + (size_t)fi * H;
    unsigned long long* xs = xsum + (size_t)fi * W;
    unsigned int mn = 0xffffffffu, mx = 0;
    unsigned long long sum = 0, cor = 0;
    const int nwarps = LR_PARTS * (LR_THREADS / 32);
    for (int y = blockIdx.x * (LR_THREADS / 32) + wid; y < H; y += nwarps) {
        const uint16_t* row = f + (size_t)y * W;
        const bool cy = (y >= 1 && y < 21) || (y >= H - 21 && y < H - 1);          // rows [1:21] and [-21:-1]
        const bool hs = y >= c.sy0 && y < c.sy1;
        unsigned long long rs = 0, strip = 0, rc = 0;
        for (int x = lane; x < W; x += 32) {
            const unsigned int v = row[x];
            mn = min(mn, v);
            mx = max(mx, v);
            rs += v;
            if (x >= c.sx0 && x < c.sx1) strip += v;
            if (cy && ((x >= 1 && x < 21) || (x >= W - 21 && x < W - 1))) rc += v;
            if (hs) atomicAdd(&xs[x], (unsigned long long)v);
        }
        sum += rs;
        cor += rc;
        strip = warp_sum(strip);
        if (lane == 0) ys[y] = strip;
    }
    mn = warp_min(mn);
    mx = warp_max(mx);
    sum = warp_sum(sum);
    cor = warp_sum(cor);
    if (lane == 0) { s_mn[wid] = mn; s_mx[wid] = mx; s_sum[wid] = sum; s_cor[wid] = cor; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < LR_THREADS / 32; k++) { mn = min(mn, s_mn[k]); mx = max(mx, s_mx[k]); }
        mn = min(mn, s_mn[0]); mx = max(mx, s_mx[0]);
        unsigned long long ts = 0, tc = 0;
        for (int k = 0; k < LR_THREADS / 32; k++) { ts += s_sum[k]; tc += s_cor[k]; }
        atomicMin(&fr[fi].mn, mn);
        atomicMax(&fr[fi].mx, mx);
        atomicAdd(&fr[fi].sum, ts);
        atomicAdd(&fr[fi].corner, tc);
    }
}

// ------------------------------------------------------------------------------------------------ field centre and widths
// _find_field_info (planar_imaging.py:1385-1420): np.mean(image[:, x0:x1], 1) and np.mean(image[y0:y1, :], 0) of the (normalised,
// possibly inverted) image, each through FWXMProfilePhysical(ground=True, normalization=BEAM_CENTER, fwxm_height=fwxm).
__global__ void __launch_bounds__(LR_THREADS)
k_lr_profile(const LrConst* __restrict__ cc, LrFrame* fr, const unsigned long long* __restrict__ ysum,
             const unsigned long long* __restrict__ xsum, char* work, size_t work_stride, int cap, int cap2) {
    __shared__ double red[40];
    __shared__ int s_small[LR_THREADS + 8];
    const LrConst& c = *cc;
    const int fi = blockIdx.x, axis = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
    const int H = c.H, W = c.W;
    LrFrame& F = fr[fi];
    // check_inversion: mean of the 4 x 400 corner pixels > mean of the frame, decided on exact integer sums (the affine map of
    // ground / normalize preserves the comparison)
    const unsigned long long npix = (unsigned long long)H * W;
    const int checked = F.corner * npix > F.sum * 1600ull ? 1 : 0;
    const int inv = checked ^ (c.p.invert ? 1 : 0);
    const unsigned int mn = F.mn, mx = F.mx;
    char* q = work + (size_t)(2 * fi + axis) * work_stride;
    auto take = [&](size_t bytes) { char* r = q; q += (bytes + 255) / 256 * 256; return r; };
    const int n = axis == 0 ? H : W;
    double* v = (double*)take(sizeof(double) * (axis == 0 ? H : W));
    PeakWork pw;
    pw.cap = cap;
    pw.prom = (double*)take(sizeof(double) * cap);
    pw.width_height = (double*)take(sizeof(double) * cap);
    pw.lip = (double*)take(sizeof(double) * cap);
    pw.rip = (double*)take(sizeof(double) * cap);
    pw.skey = (double*)take(sizeof(double) * cap2);
    pw.idx = (int*)take(sizeof(int) * cap);
    pw.lbase = (int*)take(sizeof(int) * cap);
    pw.rbase = (int*)take(sizeof(int) * cap);
    pw.flag = (int*)take(sizeof(int) * cap);
    pw.sidx = (int*)take(sizeof(int) * cap2);
    pw.s_small = s_small;
    const unsigned long long* s = axis == 0 ? ysum + (size_t)fi * H : xsum + (size_t)fi * W;
    const long long cnt = axis == 0 ? (long long)(c.sx1 - c.sx0) : (long long)(c.sy1 - c.sy0);
    const double D = (double)(mx - mn);
    for (int j = tid; j < n; j += nt) {
        const long long raw = (long long)s[j];
        double m;
        if (c.p.normalize) {
            const long long g = raw - cnt * (long long)mn;                       // sum of the grounded pixels
            const long long gi = inv ? cnt * (long long)(mx - mn) - g : g;       // -a + 1 + 0 per pixel
            m = ((double)gi / D) / (double)cnt;
        } else {
            const long long t = inv ? cnt * (long long)(mx + mn) - raw : raw;    // -v + max + min per pixel (uint16, never wraps)
            m = (double)t / (double)cnt;
        }
        v[j] = m;
    }
    __syncthreads();
    double vmin = VM_INF;
    for (int j = tid; j < n; j += nt) vmin = fmin(vmin, v[j]);
    vmin = blk_reduce<OpMin>(vmin, red);
    for (int j = tid; j < n; j += nt) v[j] = v[j] - vmin;                        // ground
    __syncthreads();
    const double fh = c.p.fwxm / 100;
    double l, r;
    int st = vm_edges(v, n, pw, &l, &r, fh);
    double center = NAN, width = NAN;
    if (!st) {
        center = fabs(r - l) / 2 + l;                                            // cached before the normalisation
        const double bcv = vm_lerp_at(v, n, center);
        __syncthreads();
        for (int j = tid; j < n; j += nt) v[j] = v[j] / bcv;                     // Normalization.BEAM_CENTER
        __syncthreads();
        st = vm_edges(v, n, pw, &l, &r, fh);
        if (!st) width = fmax(r, l) - fmin(r, l);
    }
    if (tid == 0) {
        if (axis == 0) { F.checked = checked; F.inv = inv; }
        if (st) atomicMax(&F.status, (int)EPID_LR_NO_FIELD);
        if (axis == 0) { F.cy = center; F.wy = width / c.p.dpmm; }
        else { F.cx = center; F.wx = width / c.p.dpmm; }
    }
}

// ------------------------------------------------------------------------------------------------ BB set and near-edge decisions
__device__ inline void lr_bb_position(const LrConst& c, const LrFrame& F, int k, double* px, double* py) {
    const epid_lr_params& p = c.p;
    if (p.set_mode == EPID_LR_SET_QUASAR) {
        // contrib/quasar.py:27-51: TL, BL, TR, BR offset inward from the measured field corners
        const double fs_y = F.wy / 2, fs_x = F.wx / 2, o = p.quasar_offset_mm;
        *px = k < 2 ? -fs_x + o : fs_x - o;
        *py = (k == 1 || k == 2) ? fs_y - o : -fs_y + o;
        return;
    }
    const double* set = F.large ? p.bb15_mm : p.bb_mm;
    *px = set[2 * k];
    *py = set[2 * k + 1];
}

__global__ void k_lr_plan(const LrConst* __restrict__ cc, LrFrame* fr, int n, ValueMap* vmaps, int* near_sel) {
    const int fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= n) return;
    const LrConst& c = *cc;
    LrFrame& F = fr[fi];
    vmaps[fi] = ValueMap{F.inv, F.mn, F.mx};
    int near_mask = 0;
    if (F.status == EPID_LR_OK && c.p.set_mode == EPID_LR_SET_FC2) {
        // _determine_bb_set: np.allclose(x, y, atol=10) (rtol 1e-5 of y), then the 15x15 set above 140 mm
        if (!(fabs(F.wx - F.wy) <= 10.0 + 1e-05 * fabs(F.wy))) F.status = EPID_LR_MISMATCH;
        else F.large = F.wx > 140 ? 1 : 0;
    }
    if (F.status == EPID_LR_OK) {
        const double hx = F.wx / 2, hy = F.wy / 2, t = c.p.bb_edge_threshold_mm;
        for (int k = 0; k < c.p.nbb; k++) {
            double px, py;
            lr_bb_position(c, F, k, &px, &py);
            if (fabs(px) > hx - t || fabs(py) > hy - t) near_mask |= 1 << k;
        }
    }
    F.near_mask = near_mask;
    F.near_any = near_mask != 0;
    near_sel[fi] = near_mask != 0;
}

// ------------------------------------------------------------------------------------------------ equalize_adapthist
// pixel of the once-filtered image (T = median of the mapped raw pixels) as img_as_uint sees it: rint(I * 65535) of the normalised
// float image, or the uint16 value itself without normalisation
__device__ __forceinline__ unsigned int lr_u16(const LrConst& c, const LrFrame& F, unsigned int T) {
    if (!c.p.normalize) return T;
    const double D = (double)(F.mx - F.mn);
    double a;
    if (F.inv) a = (-((double)(F.mx - T) / D) + 1.0) + 0.0;                      // invert() of the normalised image
    else a = (double)(T - F.mn) / D;
    return (unsigned int)rint(a * 65535.0);
}

// rescale_intensity(u16, out_range=(0, 2**14 - 1)) and np.round, then the histogram bin (lut = arange // (1 + 2**14 // nbins))
__device__ __forceinline__ int lr_bin(const LrConst& c, const LrFrame& F, unsigned int T) {
    const unsigned int x = lr_u16(c, F, T);
    const unsigned int a = lr_u16(c, F, F.fmn), b = lr_u16(c, F, F.fmx);
    const double imin = (double)min(a, b), imax = (double)max(a, b);
    unsigned int q;
    if (imin != imax) q = (unsigned int)rint(((double)x - imin) / (imax - imin) * 16383.0 + 0.0);
    else q = min(x, (unsigned int)(LR_NGRAY - 1));
    return (int)(q / LR_BIN);
}

__device__ __forceinline__ int lr_reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }   // np.pad 'reflect'

__global__ void __launch_bounds__(LR_THREADS)
k_lr_fminmax(const LrConst* __restrict__ cc, const uint16_t* __restrict__ filt, LrFrame* fr) {
    const LrConst& c = *cc;
    const int fi = blockIdx.y, lane = threadIdx.x & 31;
    if (!fr[fi].near_any) return;
    const size_t npx = (size_t)c.H * c.W;
    const uint16_t* f = filt + (size_t)fi * npx;
    unsigned int mn = 0xffffffffu, mx = 0;
    for (size_t i = (size_t)blockIdx.x * LR_THREADS + threadIdx.x; i < npx; i += (size_t)LR_PARTS * LR_THREADS) {
        const unsigned int v = f[i];
        mn = min(mn, v);
        mx = max(mx, v);
    }
    mn = warp_min(mn);
    mx = warp_max(mx);
    if (lane == 0) { atomicMin(&fr[fi].fmn, mn); atomicMax(&fr[fi].fmx, mx); }
}

// warp per contextual region: histogram of its k x k binned pixels, clip_histogram, map_histogram -> maps[frame][tile][256]
__global__ void __launch_bounds__(LR_THREADS)
k_lr_clahe_maps(const LrConst* __restrict__ cc, const uint16_t* __restrict__ filt, const LrFrame* __restrict__ fr,
                uint16_t* __restrict__ maps) {
    __shared__ int s_hist[LR_THREADS / 32][LR_NBINS];
    const LrConst& c = *cc;
    const int fi = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const LrFrame& F = fr[fi];
    if (!F.near_any) return;
    const int ntiles = c.nth * c.ntw;
    const int tile = blockIdx.x * (LR_THREADS / 32) + wid;
    if (tile >= ntiles) return;
    const int H = c.H, W = c.W, k = c.k;
    const uint16_t* f = filt + (size_t)fi * H * W;
    int* h = s_hist[wid];
    for (int b = lane; b < LR_NBINS; b += 32) h[b] = 0;
    __syncwarp();
    const int ti = tile / c.ntw, tj = tile - ti * c.ntw;
    for (int i = lane; i < k * k; i += 32) {
        const int ty = i / k, tx = i - ty * k;
        const int y = lr_reflect(ti * k + ty, H), x = lr_reflect(tj * k + tx, W);   // padded row k // 2 + ti k + ty
        atomicAdd(&h[lr_bin(c, F, f[(size_t)y * W + x])], 1);
    }
    __syncwarp();
    // clip_histogram: every lane owns 8 consecutive bins
    int hb[8];
#pragma unroll
    for (int e = 0; e < 8; e++) hb[e] = h[lane * 8 + e];
    const int clim = c.clim;
    long long exc = 0;
#pragma unroll
    for (int e = 0; e < 8; e++) if (hb[e] > clim) { exc += hb[e] - clim; hb[e] = clim; }
    long long n_excess = warp_sum(exc);
    const long long bin_incr = n_excess / LR_NBINS;
    const long long upper = clim - bin_incr;
    int cnt = 0;
#pragma unroll
    for (int e = 0; e < 8; e++) if (hb[e] < upper) { hb[e] += (int)bin_incr; cnt++; }
    n_excess -= (long long)warp_sum(cnt) * bin_incr;
    long long mid = 0;
#pragma unroll
    for (int e = 0; e < 8; e++) if (hb[e] >= upper && hb[e] < clim) { mid += hb[e] - clim; hb[e] = clim; }
    n_excess += warp_sum(mid);
    while (n_excess > 0) {
        const long long prev = n_excess;
        for (int index = 0; index < LR_NBINS; index++) {
            int under = 0;
#pragma unroll
            for (int e = 0; e < 8; e++) under += hb[e] < clim ? 1 : 0;
            under = warp_sum(under);
            const long long step = max(1ll, (long long)under / n_excess);
            int added = 0;
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const int b = lane * 8 + e;
                if (b >= index && (b - index) % step == 0 && hb[e] < clim) { hb[e]++; added++; }
            }
            n_excess -= warp_sum(added);
            if (n_excess <= 0) break;
        }
        if (prev == n_excess) break;
    }
    // map_histogram: int(min(cumsum * ((2**14 - 1) / (k k)) + 0, 2**14 - 1))
    int run = 0;
#pragma unroll
    for (int e = 0; e < 8; e++) run += hb[e];
    int incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
    int cum = incl - run;
    uint16_t* m = maps + ((size_t)fi * ntiles + tile) * LR_NBINS;
#pragma unroll
    for (int e = 0; e < 8; e++) {
        cum += hb[e];
        double o = (double)cum * c.map_scale + 0.0;
        o = fmin(o, (double)(LR_NGRAY - 1));
        m[lane * 8 + e] = (uint16_t)(int)o;
    }
}

// thread per pixel: the four maps around its block, weights r / k and 1 - r / k, float32 accumulation, cast back to uint16
__global__ void __launch_bounds__(LR_THREADS)
k_lr_clahe_apply(const LrConst* __restrict__ cc, const uint16_t* __restrict__ filt, const uint16_t* __restrict__ maps, LrFrame* fr,
                 uint16_t* __restrict__ out) {
    const LrConst& c = *cc;
    const int fi = blockIdx.z, lane = threadIdx.x & 31;
    LrFrame& F = fr[fi];
    if (!F.near_any) return;
    const int H = c.H, W = c.W, k = c.k;
    const int x = blockIdx.x * 32 + lane, y = blockIdx.y * (LR_THREADS / 32) + (threadIdx.x >> 5);
    unsigned int u = 0;
    const bool in = x < W && y < H;
    if (in) {
        const size_t o = (size_t)fi * H * W + (size_t)y * W + x;
        const int bin = lr_bin(c, F, filt[o]);
        const int P = y + k / 2, Q = x + k / 2;
        const int bi = P / k, r = P - bi * k, bj = Q / k, s = Q - bj * k;
        const double cr = (double)r / (double)k, cs = (double)s / (double)k;
        const uint16_t* fm = maps + (size_t)fi * c.nth * c.ntw * LR_NBINS;
        float acc = 0.0f;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int e0 = e >> 1, e1 = e & 1;
            const int ti = min(max(bi + e0 - 1, 0), c.nth - 1), tj = min(max(bj + e1 - 1, 0), c.ntw - 1);
            const double coef = (e1 ? cs : 1.0 - cs) * (e0 ? cr : 1.0 - cr);
            const double mv = (double)fm[((size_t)ti * c.ntw + tj) * LR_NBINS + bin];
            acc = acc + (float)(mv * coef);
        }
        u = (unsigned int)acc;
        out[o] = (uint16_t)u;
    }
    const unsigned int umin = warp_min(in ? u : 0xffffffffu), umax = warp_max(in ? u : 0u);
    if (lane == 0 && umin <= umax) { atomicMin(&F.umin, umin); atomicMax(&F.umax, umax); }
}

// ------------------------------------------------------------------------------------------------ locator items
// SizedDiskLocator.from_center_physical(position, (box, box), bb / 2, bb / 2) per BB (metrics/image.py:564-612 unit handling:
// expected = position * dpmm + shape / 2), Quasar's scaling search last.
__global__ void k_lr_items(const LrConst* __restrict__ cc, const LrFrame* __restrict__ fr, int n, const uint16_t* filt,
                           const uint16_t* clahe_f, const uint16_t** src, WlItemMap* maps, epid_disk_params* locs) {
    const int it = blockIdx.x * blockDim.x + threadIdx.x;
    const LrConst& c = *cc;
    if (it >= n * c.nitems) return;
    const int fi = it / c.nitems, k = it - fi * c.nitems;
    const LrFrame& F = fr[fi];
    const epid_lr_params& p = c.p;
    const double dpmm = p.dpmm;
    const size_t npx = (size_t)c.H * c.W;
    epid_disk_params& L = locs[it];
    memset(&L, 0, sizeof(L));
    L.dpmm = dpmm;
    L.invert = 1;
    L.conditions = 31;                 // DEFAULT_CONDITIONS (metrics/features.py)
    WlItemMap m;
    m.status = F.status == EPID_LR_OK ? EPID_WL_OK : EPID_WL_NO_BB;
    if (p.normalize) { m.mn = F.mn; m.D = F.mx - F.mn; }
    else { m.mn = 0; m.D = 1; }
    src[it] = filt + (size_t)fi * npx;
    if (k < p.nbb) {
        double px = 0, py = 0;
        if (F.status == EPID_LR_OK) lr_bb_position(c, F, k, &px, &py);
        L.expected_x = px * dpmm + (double)c.W / 2;
        L.expected_y = py * dpmm + (double)c.H / 2;
        L.window_w = L.window_h = p.bb_box_mm * dpmm;
        L.radius_mm = p.bb_size_mm / 2;
        L.tolerance_mm = p.bb_size_mm / 2;
        L.min_separation_px = 5.0 * dpmm;
        L.max_number = 1;
        if (F.near_mask & (1 << k)) {
            src[it] = clahe_f + (size_t)fi * npx;
            m.mn = F.umin;
            m.D = F.umax > F.umin ? F.umax - F.umin : 1;      // a flat result: the locator's stretch finds nothing either way
        }
    } else {
        // _detect_scaling_centers: 35 mm window about the image centre, exactly 5 disks at least 4 mm apart
        L.expected_x = 0.0 * dpmm + (double)c.W / 2;
        L.expected_y = 0.0 * dpmm + (double)c.H / 2;
        L.window_w = L.window_h = 35.0 * dpmm;
        L.radius_mm = p.bb_size_mm / 2;
        L.tolerance_mm = p.bb_size_mm / 2;
        L.min_separation_px = 4.0 * dpmm;
        L.max_number = EPID_LR_SCALING;
    }
    maps[it] = m;
}

__global__ void k_lr_finalize(const LrConst* __restrict__ cc, const LrFrame* __restrict__ fr, int n, const epid_disk_result* __restrict__ dres,
                              epid_lr_result* __restrict__ res) {
    const int fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= n) return;
    const LrConst& c = *cc;
    const LrFrame& F = fr[fi];
    epid_lr_result& R = res[fi];
    memset(&R, 0, sizeof(R));
    R.status = F.status;
    R.inverted = F.checked;
    R.large_set = F.large;
    R.near_edge_mask = F.near_mask;
    R.field_center_x = F.cx;
    R.field_center_y = F.cy;
    R.field_width_x_mm = F.wx;
    R.field_width_y_mm = F.wy;
    if (R.status == EPID_LR_OK) {
        for (int k = 0; k < c.nitems; k++) {
            const epid_disk_result& D = dres[fi * c.nitems + k];
            const int need = k < c.p.nbb ? 1 : EPID_LR_SCALING;
            const int found = D.status == EPID_WL_OK ? D.n_points : 0;
            if (D.status == EPID_WL_CAPACITY) { R.status = EPID_LR_CAPACITY; R.failed_bb = k; break; }
            if (found < need) { R.status = EPID_LR_NO_BB; R.failed_bb = k; R.n_found = found; break; }
            if (k < c.p.nbb) { R.bb_x[k] = D.x[0]; R.bb_y[k] = D.y[0]; }
            else {
                R.n_scaling = found;
                for (int j = 0; j < found && j < EPID_LR_SCALING; j++) { R.scaling_x[j] = D.x[j]; R.scaling_y[j] = D.y[j]; }
            }
        }
    }
}

// host destinations of the diagnostic read-back (epid_lightrad_stages); epid_lightrad_analyze passes none
struct LrTap {
    uint16_t* filtered;
    uint16_t* equalised;
    uint16_t* equalised_filtered;
    LrFrame* frames;
};

}  // namespace epid

using namespace epid;

static int32_t lightrad_run(epid_ctx* ctx, const epid_batch* frames, const epid_lr_params* p, epid_lr_result* results,
                            const LrTap* tap) {
    EPID_REQUIRE(ctx && frames && p && results, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(frames->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "light/rad frames must be uint16");
    EPID_REQUIRE(p->dpmm > 0 && p->bb_size_mm > 0 && p->bb_box_mm > 0 && p->strip_width_mm > 0, EPID_ERR_INVALID, "bad geometry");
    EPID_REQUIRE(p->nbb >= 1 && p->nbb <= EPID_LR_MAX_BB, EPID_ERR_INVALID, "1..%d BBs", EPID_LR_MAX_BB);
    EPID_REQUIRE(p->set_mode != EPID_LR_SET_QUASAR || p->nbb == 4, EPID_ERR_INVALID, "the Quasar set has 4 BBs");
    EPID_REQUIRE(p->fwxm >= 0 && p->fwxm <= 100, EPID_ERR_INVALID, "fwxm must be between 0 and 100");
    const int n = frames->n, H = frames->h, W = frames->w;
    EPID_REQUIRE(H >= 64 && W >= 64, EPID_ERR_UNSUPPORTED, "frames smaller than 64 x 64");
    EPID_REQUIRE(p->clahe_kernel >= 1 && p->clahe_kernel < (H < W ? H : W), EPID_ERR_INVALID, "CLAHE kernel size %d", p->clahe_kernel);
    EPID_CUDA(cudaSetDevice(ctx->device));
    LrConst hc;
    memset(&hc, 0, sizeof(hc));
    hc.p = *p;
    hc.H = H;
    hc.W = W;
    // _find_field_info: int(centre -+ strip / 2 * dpmm) with image.center = shape / 2 - 0.5
    const double sw = p->strip_width_mm / 2 * p->dpmm;
    hc.sx0 = (int)((double)W / 2 - 0.5 - sw); hc.sx1 = (int)((double)W / 2 - 0.5 + sw);
    hc.sy0 = (int)((double)H / 2 - 0.5 - sw); hc.sy1 = (int)((double)H / 2 - 0.5 + sw);
    EPID_REQUIRE(hc.sx0 >= 0 && hc.sx1 <= W && hc.sx1 > hc.sx0 && hc.sy0 >= 0 && hc.sy1 <= H && hc.sy1 > hc.sy0, EPID_ERR_INVALID,
                 "strip outside the frame");
    const int k = p->clahe_kernel;
    hc.k = k;
    // np.pad(image, [[k // 2, (k - s % k) % k + ceil(k / 2)]]): the padded length is a multiple of k; one region fewer than blocks
    hc.nth = (H + k / 2 + (k - H % k) % k + (k + 1) / 2) / k - 1;
    hc.ntw = (W + k / 2 + (k - W % k) % k + (k + 1) / 2) / k - 1;
    const double clim = 0.01 * (double)(k * k);
    hc.clim = clim < 1 ? 1 : (int)clim;
    hc.map_scale = (double)(LR_NGRAY - 1) / (double)(k * k);
    hc.nitems = p->nbb + (p->scaling ? 1 : 0);
    const int chunk = n < 64 ? n : 64;
    const int cap = (H > W ? H : W) / 2 + 1;
    int cap2 = 1;
    while (cap2 < (H > W ? H : W)) cap2 <<= 1;
    auto rup = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t work_stride = rup(sizeof(double) * (H > W ? H : W)) + 4 * rup(sizeof(double) * cap) + rup(sizeof(double) * cap2) +
                               4 * rup(sizeof(int) * cap) + rup(sizeof(int) * cap2);
    const size_t npx = (size_t)H * W;
    const int nit = chunk * hc.nitems;
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += rup(b); return r; };
    const size_t o_cst = sz(sizeof(LrConst)), o_fr = sz(sizeof(LrFrame) * chunk), o_ys = sz(sizeof(unsigned long long) * chunk * (size_t)H);
    const size_t o_xs = sz(sizeof(unsigned long long) * chunk * (size_t)W), o_wk = sz(work_stride * 2 * chunk);
    const size_t o_vm = sz(sizeof(ValueMap) * chunk), o_sel = sz(sizeof(int) * chunk);
    const size_t o_refs = sz(sizeof(FrameRef) * 4 * chunk);
    const size_t o_filt = sz(sizeof(uint16_t) * npx * chunk), o_eq = sz(sizeof(uint16_t) * npx * chunk), o_eqf = sz(sizeof(uint16_t) * npx * chunk);
    const size_t o_maps = sz(sizeof(uint16_t) * (size_t)hc.nth * hc.ntw * LR_NBINS * chunk);
    const size_t o_src = sz(sizeof(uint16_t*) * nit), o_imap = sz(sizeof(WlItemMap) * nit), o_loc = sz(sizeof(epid_disk_params) * nit);
    const size_t o_dres = sz(sizeof(epid_disk_result) * nit), o_res = sz(sizeof(epid_lr_result) * chunk);
    const size_t o_items = sz(disk_items_scratch_bytes(nit));
    int rc = ensure_scratch(ctx, o);
    if (rc != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    cudaStream_t st = ctx->stream;
    LrConst* d_cst = (LrConst*)(base + o_cst);
    LrFrame* d_fr = (LrFrame*)(base + o_fr);
    FrameRef* refs = (FrameRef*)(base + o_refs);
    uint16_t* d_filt = (uint16_t*)(base + o_filt);
    uint16_t* d_eq = (uint16_t*)(base + o_eq);
    uint16_t* d_eqf = (uint16_t*)(base + o_eqf);
    const double max_window = (p->scaling ? fmax(35.0, p->bb_box_mm) : p->bb_box_mm) * p->dpmm;
    EPID_CUDA(cudaMemcpyAsync(d_cst, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    for (int c0 = 0; c0 < n; c0 += chunk) {
        const int cn = n - c0 < chunk ? n - c0 : chunk;
        const uint16_t* d_frames = (const uint16_t*)frames->dptr + (size_t)c0 * npx;
        EPID_CUDA(cudaMemsetAsync(base + o_xs, 0, sizeof(unsigned long long) * cn * (size_t)W, st));
        k_lr_init<<<(cn + 127) / 128, 128, 0, st>>>(d_fr, cn);
        k_lr_front<<<dim3(LR_PARTS, cn), LR_THREADS, 0, st>>>(d_cst, d_frames, d_fr, (unsigned long long*)(base + o_ys),
                                                             (unsigned long long*)(base + o_xs));
        k_lr_profile<<<dim3(cn, 2), LR_THREADS, 0, st>>>(d_cst, d_fr, (const unsigned long long*)(base + o_ys),
                                                         (const unsigned long long*)(base + o_xs), base + o_wk, work_stride, cap, cap2);
        k_lr_plan<<<(cn + 127) / 128, 128, 0, st>>>(d_cst, d_fr, cn, (ValueMap*)(base + o_vm), (int*)(base + o_sel));
        ctx->launches += 4;
        // image.filter(size=3, kind="median") of the mapped frame (:1433)
        launch_refs_from_batch(ctx, st, d_frames, cn, H, W, 0, 0, refs);
        launch_refs_from_batch(ctx, st, d_filt, cn, H, W, 0, 0, refs + chunk);
        launch_refs_from_batch(ctx, st, d_eq, cn, H, W, 0, 0, refs + 2 * chunk);
        launch_refs_from_batch(ctx, st, d_eqf, cn, H, W, 0, 0, refs + 3 * chunk);
        rc = launch_median_u16(ctx, st, refs, refs + chunk, (const ValueMap*)(base + o_vm), nullptr, cn, H, W, 3);
        if (rc != EPID_OK) return rc;
        // equalize_adapthist + the second median, frames with a near-edge BB only
        k_lr_fminmax<<<dim3(LR_PARTS, cn), LR_THREADS, 0, st>>>(d_cst, d_filt, d_fr);
        const int ntiles = hc.nth * hc.ntw;
        k_lr_clahe_maps<<<dim3((ntiles + LR_THREADS / 32 - 1) / (LR_THREADS / 32), cn), LR_THREADS, 0, st>>>(d_cst, d_filt, d_fr,
                                                                                                          (uint16_t*)(base + o_maps));
        k_lr_clahe_apply<<<dim3((W + 31) / 32, (H + LR_THREADS / 32 - 1) / (LR_THREADS / 32), cn), LR_THREADS, 0, st>>>(
            d_cst, d_filt, (const uint16_t*)(base + o_maps), d_fr, d_eq);
        ctx->launches += 3;
        rc = launch_median_u16(ctx, st, refs + 2 * chunk, refs + 3 * chunk, nullptr, (const int*)(base + o_sel), cn, H, W, 3);
        if (rc != EPID_OK) return rc;
        // the windowed locator per BB (and the Quasar scaling search)
        const int ni = cn * hc.nitems;
        k_lr_items<<<(ni + 127) / 128, 128, 0, st>>>(d_cst, d_fr, cn, d_filt, d_eqf, (const uint16_t**)(base + o_src),
                                                     (WlItemMap*)(base + o_imap), (epid_disk_params*)(base + o_loc));
        ctx->launches += 1;
        EPID_CUDA(cudaMemsetAsync(base + o_dres, 0, sizeof(epid_disk_result) * ni, st));
        rc = launch_disk_items(ctx, st, base + o_items, ni, H, W, p->dpmm, max_window, (const uint16_t* const*)(base + o_src),
                               (const WlItemMap*)(base + o_imap), (const epid_disk_params*)(base + o_loc), (epid_disk_result*)(base + o_dres));
        if (rc != EPID_OK) return rc;
        k_lr_finalize<<<(cn + 127) / 128, 128, 0, st>>>(d_cst, d_fr, cn, (const epid_disk_result*)(base + o_dres), (epid_lr_result*)(base + o_res));
        ctx->launches += 1;
        EPID_CUDA(cudaGetLastError());
        EPID_CUDA(cudaMemcpyAsync(results + c0, base + o_res, sizeof(epid_lr_result) * cn, cudaMemcpyDeviceToHost, st));
        if (tap) {
            // stream order: the copies finish before the next chunk reuses the planes
            const size_t pb = sizeof(uint16_t) * npx * cn;
            EPID_CUDA(cudaMemcpyAsync(tap->filtered + (size_t)c0 * npx, d_filt, pb, cudaMemcpyDeviceToHost, st));
            EPID_CUDA(cudaMemcpyAsync(tap->equalised + (size_t)c0 * npx, d_eq, pb, cudaMemcpyDeviceToHost, st));
            EPID_CUDA(cudaMemcpyAsync(tap->equalised_filtered + (size_t)c0 * npx, d_eqf, pb, cudaMemcpyDeviceToHost, st));
            EPID_CUDA(cudaMemcpyAsync(tap->frames + c0, d_fr, sizeof(LrFrame) * cn, cudaMemcpyDeviceToHost, st));
        }
    }
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("light/rad pipeline failed: %s", cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    return EPID_OK;
}

extern "C" int32_t epid_lightrad_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_lr_params* p, epid_lr_result* results) {
    return lightrad_run(ctx, frames, p, results, nullptr);
}

extern "C" int32_t epid_lightrad_stages(epid_ctx* ctx, const epid_batch* frames, const epid_lr_params* p, epid_lr_result* results,
                                        uint16_t* filtered, uint16_t* equalised, uint16_t* equalised_filtered, int64_t* info) {
    EPID_REQUIRE(frames && filtered && equalised && equalised_filtered && info, EPID_ERR_INVALID, "NULL argument");
    std::vector<LrFrame> fr((size_t)(frames->n > 0 ? frames->n : 0));
    const LrTap tap{filtered, equalised, equalised_filtered, fr.data()};
    const int32_t rc = lightrad_run(ctx, frames, p, results, &tap);
    if (rc != EPID_OK) return rc;
    for (size_t i = 0; i < fr.size(); i++) {
        const LrFrame& F = fr[i];
        const int64_t row[EPID_LR_INFO] = {F.mn, F.mx, (int64_t)F.sum, (int64_t)F.corner, F.checked, F.inv, F.near_mask,
                                           F.fmn, F.fmx, F.umin, F.umax};
        memcpy(info + i * EPID_LR_INFO, row, sizeof(row));
    }
    return EPID_OK;
}
