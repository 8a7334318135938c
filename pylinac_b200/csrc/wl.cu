// Batched per-image (2-D) Winston-Lutz analysis on the GPU.  One result per frame; frames never leave HBM between stages.
//
// Reference path reproduced (pylinac v3.46.0):
//   WLBaseImage.analyze / _clean_edges / find_field_centroids / find_bb_centroids / find_bb_matches   winston_lutz.py:668-829, 1109-1133
//   WinstonLutz2D.analyze / cax2bb_* / cax2epid_*                                                       winston_lutz.py:1137-1231
//   SizedDiskLocator.calculate (from_center_physical)                                                   metrics/image.py:526-612, 661-667
//   find_features / deduplicate_points_and_boundaries                                                   metrics/utils.py:14-37, 66-190
//   predicates is_right_size_bb / is_round / is_right_circumference / is_symmetric / is_solid           metrics/features.py:7-68
//   BaseImage.check_inversion_by_histogram / crop / ground / normalize / as_binary                      core/image.py:714-866, 899-926
//   array_utils.invert / stretch                                                                        core/array_utils.py:75-77, 142-168
// Third-party functions restated: scipy.ndimage.binary_fill_holes (4-connected flood of the background from the border),
// center_of_mass; skimage.measure.label(connectivity=1) (union-find, labels in raster order of the first pixel),
// segmentation.clear_border, regionprops bbox / area / area_filled / perimeter (4-neighbourhood border, 3x3 weighted
// convolution, weights 1 / sqrt2 / (1+sqrt2)/2) / solidity (pixel centres inside the convex hull of the pixels' diamond offsets) /
// centroid_weighted.  skimage is absent from the build container: perimeter and convex area follow the published algorithms and
// agree with oracle/skimage_shim.py; that boundary is UNPINNED against skimage itself (SURVEY.md section 8c).
//
// Exactness: after the histogram inversion check, the edge clean-up, ground and normalize the image is I = g / D with g an
// integer map of the uint16 frame (g = T(v) - min, T(v) = v or max0 + min0 - v).  Percentiles are exact order statistics read from
// a 65536-bin histogram that is updated incrementally when _clean_edges crops a 2-pixel ring; thresholds on I are turned into
// integer thresholds on g; the BB sample repeats the reference's fp64 operation order (invert, stretch) pixel by pixel.
//
// Stages:
//   k_wl_hist    exact 65536-bin histogram of every frame (shared-memory bin cache of stats.cuh)
//   k_wl_front   CTA per frame: inversion decision, _clean_edges loop (percentiles from the histogram, ring min / max, ring
//                removal), ground / normalize constants, field threshold
//   k_wl_field   CTA per frame: bounding box of the thresholded field, fill holes inside it, centre of mass
//   k_wl_bb      CTA per frame: BB window -> stretched sample -> <= 50 thresholds { union-find labelling, region properties,
//                predicates } -> weighted centroid(s); field / BB matching and the result row
#include <cmath>

#include "pf_common.cuh"
#include "ccl.cuh"
#include "wl.cuh"

namespace epid {

constexpr int WL_THREADS = 256;
constexpr int WL_WARPS = WL_THREADS / 32;
constexpr int WL_MAXC = 8192;          // components per threshold with accumulators (HBM scratch)
constexpr int WL_TILE = 96;            // candidate region tile (bbox + margin) edge
constexpr int WL_MAXPTS = 8;           // detected BB points per image
constexpr int WL_MAXWIN = 224;         // BB window edge in pixels

struct WlConst {
    epid_wl_params p;
    int H, W;
    size_t field_tile_cap;             // bytes available for the field tile in k_wl_field's dynamic shared memory
    int win_edge;                      // largest BB window edge of this launch: the union-find forest holds win_edge^2 ints
    // stand-alone disk locator (SizedDiskRegion / SizedDiskLocator, metrics/image.py:402-667): the BB search of k_wl_bb on a raw frame
    int loc_mode;                      // 0: Winston-Lutz flow, 1: epid_disk_locate
    epid_disk_params loc;
};

struct WlFrame {
    int status;
    int flip;                          // pixels are read as T(v) = flip ? S - v : v
    uint32_t S;                        // max0 + min0 of the uncropped frame
    int crop;                          // pixels removed from every edge by _clean_edges
    int h, w;                          // cropped shape
    uint32_t mn, D;                    // ground / normalize: I = (T(v) - mn) / D
    uint32_t g_field;                  // field mask: g >= g_field  <=>  I >= (p99.9 - p5) / 2 + p5
    double field_x, field_y;
    int by0, by1, bx0, bx1;            // bounding box of the thresholded field (k_wl_bbox)
};

__device__ __forceinline__ uint32_t wl_T(const WlFrame& f, uint32_t v) { return f.flip ? f.S - v : v; }

// ------------------------------------------------------------------------------------------------ histogram
constexpr int WL_HPARTS = 8;           // CTAs per frame
static_assert(WL_THREADS == HIST_RANK_THREADS, "k_wl_front runs hist_rank_search with all its threads");

// Exact histogram.  A CTA streams 1/8 of a frame with 16-byte loads and counts it through the bin cache of stats.cuh.
__global__ void __launch_bounds__(256)
k_wl_hist(const uint16_t* __restrict__ base, int H, int W, uint32_t* __restrict__ hist) {
    __shared__ HistCache s_cache;
    const int fi = blockIdx.y;
    const uint16_t* f = base + (size_t)fi * H * W;
    uint32_t* h = hist + (size_t)fi * 65536;
    const int lane = threadIdx.x & 31;
    hist_cache_init(s_cache);
    __syncthreads();
    const size_t npx = (size_t)H * W;
    const size_t per = ((npx + WL_HPARTS - 1) / WL_HPARTS + 7) & ~(size_t)7;
    const size_t p0 = (size_t)blockIdx.x * per, p1 = p0 + per < npx ? p0 + per : npx;
    // head up to the first 16-byte boundary, vector body, tail
    const size_t mis = ((reinterpret_cast<uintptr_t>(f + p0) >> 1) & 7);
    const size_t v0 = p0 + ((8 - mis) & 7) < p1 ? p0 + ((8 - mis) & 7) : p1;
    const size_t nvec = (p1 - v0) >> 3;
    if (threadIdx.x < 32) hist_cache_add(s_cache, h, p0 + lane < v0 ? f[p0 + lane] : 0u, p0 + lane < v0);
    const size_t nvec32 = (nvec + 31) & ~(size_t)31;            // every lane of a warp takes the same number of trips
    for (size_t k = threadIdx.x; k < ((nvec32 + 255) & ~(size_t)255); k += 256) {
        const bool in = k < nvec;
        uint4 q = make_uint4(0, 0, 0, 0);
        if (in) q = ldg_stream16(f + v0 + k * 8);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int t = 0; t < 4; t++) {
            hist_cache_add(s_cache, h, w[t] & 0xffffu, in);
            hist_cache_add(s_cache, h, w[t] >> 16, in);
        }
    }
    const size_t t0 = v0 + nvec * 8;
    if (threadIdx.x < 32) hist_cache_add(s_cache, h, t0 + lane < p1 ? f[t0 + lane] : 0u, t0 + lane < p1);
    __syncthreads();
    hist_cache_flush(s_cache, h);
}

// ------------------------------------------------------------------------------------------------ front
struct WlScan {
    HistRanks q;                       // values of up to 8 raw order statistics + first / last non-empty bin (hist_rank_search)
    uint32_t ranks[8];
    double d[WL_WARPS];
    uint32_t u[2 * WL_WARPS];
};

__global__ void __launch_bounds__(WL_THREADS)
k_wl_front(const WlConst* __restrict__ cc, const uint16_t* __restrict__ base, uint32_t* __restrict__ hist_all, WlFrame* wf) {
    __shared__ WlScan s;
    __shared__ int s_noisy;
    const WlConst& c = *cc;
    const int fi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int H = c.H, W = c.W;
    const uint16_t* f = base + (size_t)fi * H * W;
    uint32_t* hist = hist_all + (size_t)fi * 65536;
    const volatile uint32_t* hist_v = hist;   // the searches read the histogram that _clean_edges updates in this kernel
    WlFrame& F = wf[fi];
    // ---- check_inversion_by_histogram((0.01, 50, 99.99)) (core/image.py:899-926)
    uint32_t n = (uint32_t)H * (uint32_t)W;
    if (tid == 0) {
        const double qs[3] = {0.01, 50.0, 99.99};
        for (int k = 0; k < 3; k++) {
            const PctPlan pp = pct_plan((int)n, qs[k]);
            s.ranks[2 * k] = pp.prev;
            s.ranks[2 * k + 1] = pp.next;
        }
    }
    __syncthreads();
    hist_rank_search(hist_v, s.ranks, 6, s.q);
    int flip = 0;
    uint32_t S = 0;
    {
        const double qs[3] = {0.01, 50.0, 99.99};
        double p[3];
        for (int k = 0; k < 3; k++) p[k] = np_lerp((double)s.q.values[2 * k], (double)s.q.values[2 * k + 1], pct_plan((int)n, qs[k]).gamma);
        flip = fabs(p[1] - p[0]) > fabs(p[1] - p[2]) ? 1 : 0;
        S = s.q.first + s.q.last;                      // invert(): -a + max + min of the uncropped frame
    }
    __syncthreads();
    if (s.q.first == s.q.last) {
        if (tid == 0) { F.status = EPID_WL_FLAT_IMAGE; F.flip = 0; F.S = 0; F.crop = 0; F.h = H; F.w = W; F.mn = 0; F.D = 0; F.g_field = 0; F.by0 = H; F.by1 = -1; F.bx0 = W; F.bx1 = -1; }
        return;
    }
    // ---- _clean_edges(window_size=2) (winston_lutz.py:1109-1133)
    int crop = 0;
    double safety = (double)(H < W ? H : W) / 10;
    while (safety > 0) {
        const int h = H - 2 * crop, w = W - 2 * crop;
        if (h <= 4 || w <= 4) break;
        n = (uint32_t)h * (uint32_t)w;
        const PctPlan p5 = pct_plan((int)n, 5.0), p9 = pct_plan((int)n, 99.5);
        const uint32_t r5a = p5.prev, r5b = p5.next, r9a = p9.prev, r9b = p9.next;
        const double g5 = p5.gamma, g9 = p9.gamma;
        if (tid == 0) {
            // T-domain rank k = raw rank n - 1 - k when flipped (T is decreasing)
            s.ranks[0] = flip ? n - 1 - r5a : r5a; s.ranks[1] = flip ? n - 1 - r5b : r5b;
            s.ranks[2] = flip ? n - 1 - r9a : r9a; s.ranks[3] = flip ? n - 1 - r9b : r9b;
        }
        __syncthreads();
        hist_rank_search(hist_v, s.ranks, 4, s.q);
        const double t5a = flip ? (double)(S - s.q.values[0]) : (double)s.q.values[0], t5b = flip ? (double)(S - s.q.values[1]) : (double)s.q.values[1];
        const double t9a = flip ? (double)(S - s.q.values[2]) : (double)s.q.values[2], t9b = flip ? (double)(S - s.q.values[3]) : (double)s.q.values[3];
        const double near_min = np_lerp(t5a, t5b, g5), near_max = np_lerp(t9a, t9b, g9);
        const double img_range = near_max - near_min;
        // min / max of the 2-pixel border of the current view (T domain)
        uint32_t emin = 0xffffffffu, emax = 0;
        const int ring = 2 * 2 * w + 2 * 2 * (h - 4);
        for (int i = tid; i < ring; i += WL_THREADS) {
            int y, x;
            if (i < 2 * w) { y = i / w; x = i - y * w; }
            else if (i < 4 * w) { const int j = i - 2 * w; y = h - 2 + j / w; x = j % w; }
            else { const int j = i - 4 * w; y = 2 + j / 4; const int k = j & 3; x = k < 2 ? k : w - 4 + k; }
            const uint32_t v = f[(size_t)(y + crop) * W + (x + crop)];
            const uint32_t t = flip ? S - v : v;
            emin = min(emin, t);
            emax = max(emax, t);
        }
        emin = warp_min(emin);
        emax = warp_max(emax);
        if (lane == 0) { s.u[wid] = emin; s.u[WL_WARPS + wid] = emax; }
        __syncthreads();
        if (tid == 0) {
            uint32_t a = s.u[0], b = s.u[WL_WARPS];
            for (int k = 1; k < WL_WARPS; k++) { a = min(a, s.u[k]); b = max(b, s.u[WL_WARPS + k]); }
            const bool too_low = (double)a < (near_min - img_range / 10);
            const bool too_high = (double)b > (near_max + img_range / 10);
            s_noisy = (too_low || too_high) ? 1 : 0;
        }
        __syncthreads();
        if (!s_noisy) break;
        // crop(2): remove the ring from the histogram
        for (int i = tid; i < ring; i += WL_THREADS) {
            int y, x;
            if (i < 2 * w) { y = i / w; x = i - y * w; }
            else if (i < 4 * w) { const int j = i - 2 * w; y = h - 2 + j / w; x = j % w; }
            else { const int j = i - 4 * w; y = 2 + j / 4; const int k = j & 3; x = k < 2 ? k : w - 4 + k; }
            atomicSub(&hist[f[(size_t)(y + crop) * W + (x + crop)]], 1u);
        }
        __threadfence();
        __syncthreads();
        crop += 2;
        safety -= 1;
    }
    // ---- ground() / normalize() constants and the field threshold (winston_lutz.py:711-712, 764-780)
    const int h = H - 2 * crop, w = W - 2 * crop;
    n = (uint32_t)h * (uint32_t)w;
    const PctPlan p5 = pct_plan((int)n, 5.0), p9 = pct_plan((int)n, 99.9);
    const uint32_t r5a = p5.prev, r5b = p5.next, r9a = p9.prev, r9b = p9.next;
    const double g5 = p5.gamma, g9 = p9.gamma;
    if (tid == 0) {
        s.ranks[0] = flip ? n - 1 - r5a : r5a; s.ranks[1] = flip ? n - 1 - r5b : r5b;
        s.ranks[2] = flip ? n - 1 - r9a : r9a; s.ranks[3] = flip ? n - 1 - r9b : r9b;
    }
    __syncthreads();
    hist_rank_search(hist_v, s.ranks, 4, s.q);
    if (tid == 0) {
        const uint32_t tmin = flip ? S - s.q.last : s.q.first, tmax = flip ? S - s.q.first : s.q.last;
        const uint32_t D = tmax - tmin;
        F.status = D == 0 ? EPID_WL_FLAT_IMAGE : EPID_WL_OK;
        F.flip = flip;
        F.S = S;
        F.crop = crop;
        F.h = h;
        F.w = w;
        F.mn = tmin;
        F.D = D;
        F.g_field = 0;
        F.by0 = h; F.by1 = -1; F.bx0 = w; F.bx1 = -1;
        if (D) {
            double v[4];
            for (int k = 0; k < 4; k++) {
                const uint32_t t = flip ? S - s.q.values[k] : s.q.values[k];
                v[k] = (double)(t - tmin) / (double)D;              // normalized pixel values
            }
            const double pmin = np_lerp(v[0], v[1], g5), pmax = np_lerp(v[2], v[3], g9);
            const double thr = (pmax - pmin) / 2 + pmin;
            // as_binary(thr): I >= thr  <=>  g >= g*, g* = smallest integer with (double)g / D >= thr (I is monotone in g)
            uint32_t lo = 0, hi = D + 1;
            while (lo < hi) {
                const uint32_t mid = lo + (hi - lo) / 2;
                if ((double)mid / (double)D >= thr) hi = mid; else lo = mid + 1;
            }
            F.g_field = lo;
        }
    }
}

// ------------------------------------------------------------------------------------------------ field centroid
// flood the complement of `mask` from the tile border (4-connectivity), row / column sweeps until nothing changes:
// tile[i]: 1 = mask, 0 = background not yet reached, 2 = background connected to the border
__device__ inline void wl_flood_outside(unsigned char* tile, int th, int tw) {
    const int tid = threadIdx.x;
    for (int i = tid; i < th * tw; i += WL_THREADS) {
        const int y = i / tw, x = i - y * tw;
        if ((y == 0 || x == 0 || y == th - 1 || x == tw - 1) && tile[i] == 0) tile[i] = 2;
    }
    __syncthreads();
    while (true) {
        int changed = 0;
        for (int y = tid; y < th; y += WL_THREADS) {
            unsigned char* r = tile + (size_t)y * tw;
            for (int x = 1; x < tw; x++) if (r[x] == 0 && r[x - 1] == 2) { r[x] = 2; changed = 1; }
            for (int x = tw - 2; x >= 0; x--) if (r[x] == 0 && r[x + 1] == 2) { r[x] = 2; changed = 1; }
        }
        __syncthreads();
        for (int x = tid; x < tw; x += WL_THREADS) {
            for (int y = 1; y < th; y++) if (tile[(size_t)y * tw + x] == 0 && tile[(size_t)(y - 1) * tw + x] == 2) { tile[(size_t)y * tw + x] = 2; changed = 1; }
            for (int y = th - 2; y >= 0; y--) if (tile[(size_t)y * tw + x] == 0 && tile[(size_t)(y + 1) * tw + x] == 2) { tile[(size_t)y * tw + x] = 2; changed = 1; }
        }
        if (!__syncthreads_or(changed)) break;
    }
}

constexpr int WL_BBOX_PARTS = 16;      // CTAs per frame in the bounding-box pass

// bounding box of the field mask (I >= threshold), rows dealt to warps, coalesced 2-byte loads, one atomic per warp
__global__ void __launch_bounds__(WL_THREADS)
k_wl_bbox(const WlConst* __restrict__ cc, const uint16_t* __restrict__ base, WlFrame* wf) {
    const WlConst& c = *cc;
    const int fi = blockIdx.y, lane = threadIdx.x & 31;
    WlFrame& F = wf[fi];
    if (F.status != EPID_WL_OK || c.p.open_field) return;
    const int W = c.W;
    const uint16_t* f = base + (size_t)fi * c.H * W;
    const int h = F.h, w = F.w, crop = F.crop;
    const uint32_t gth = F.g_field, mn = F.mn, S = F.S;
    const int flip = F.flip;
    int y0 = h, y1 = -1, x0 = w, x1 = -1;
    const int nwarps = WL_BBOX_PARTS * WL_WARPS;
    for (int y = blockIdx.x * WL_WARPS + (threadIdx.x >> 5); y < h; y += nwarps) {
        const uint16_t* row = f + (size_t)(y + crop) * W + crop;
        for (int x = lane; x < w; x += 32) {
            const uint32_t v = row[x];
            const uint32_t g = (flip ? S - v : v) - mn;
            if (g >= gth) { y0 = min(y0, y); y1 = max(y1, y); x0 = min(x0, x); x1 = max(x1, x); }
        }
    }
    y0 = warp_min(y0); y1 = warp_max(y1); x0 = warp_min(x0); x1 = warp_max(x1);
    if (lane == 0 && y1 >= 0) { atomicMin(&F.by0, y0); atomicMax(&F.by1, y1); atomicMin(&F.bx0, x0); atomicMax(&F.bx1, x1); }
}

__global__ void __launch_bounds__(WL_THREADS)
k_wl_field(const WlConst* __restrict__ cc, const uint16_t* __restrict__ base, WlFrame* wf) {
    extern __shared__ __align__(16) unsigned char tile[];
    __shared__ unsigned long long s_sum[3];
    const WlConst& c = *cc;
    const int fi = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    WlFrame& F = wf[fi];
    if (F.status != EPID_WL_OK) return;
    const int H = c.H, W = c.W;
    const uint16_t* f = base + (size_t)fi * H * W;
    const int h = F.h, w = F.w, crop = F.crop;
    if (c.p.open_field) {      // find_field_centroids(is_open_field=True): the CAX (winston_lutz.py:764-767)
        if (tid == 0) { F.field_x = (double)w / 2 - 0.5; F.field_y = (double)h / 2 - 0.5; }
        return;
    }
    const uint32_t gth = F.g_field, mn = F.mn;
    if (tid == 0) { s_sum[0] = s_sum[1] = s_sum[2] = 0; }
    __syncthreads();
    const int y0 = F.by0, y1 = F.by1, x0 = F.bx0, x1 = F.bx1;      // k_wl_bbox
    if (y1 < 0) { if (tid == 0) F.status = EPID_WL_NO_FIELD; return; }     // center_of_mass of nothing: nan in the reference
    // tile = bounding box + 1 pixel of margin (the margin is background reachable from the image border or is outside the image)
    const int th = y1 - y0 + 3, tw = x1 - x0 + 3;
    if ((size_t)th * tw > c.field_tile_cap) { if (tid == 0) F.status = EPID_WL_CAPACITY; return; }
    for (int i = tid; i < th * tw; i += WL_THREADS) {
        const int ty = i / tw, tx = i - ty * tw;
        const int y = y0 - 1 + ty, x = x0 - 1 + tx;
        unsigned char m = 0;
        if (y >= 0 && y < h && x >= 0 && x < w) m = (wl_T(F, f[(size_t)(y + crop) * W + (x + crop)]) - mn) >= gth ? 1 : 0;
        tile[i] = m;
    }
    __syncthreads();
    wl_flood_outside(tile, th, tw);
    // ndimage.center_of_mass(binary_fill_holes(mask)): exact integer coordinate sums / count
    unsigned long long sy = 0, sx = 0, cnt = 0;
    for (int i = tid; i < th * tw; i += WL_THREADS) {
        if (tile[i] != 2) {
            const int ty = i / tw, tx = i - ty * tw;
            sy += (unsigned long long)(y0 - 1 + ty);
            sx += (unsigned long long)(x0 - 1 + tx);
            cnt++;
        }
    }
    sy = warp_sum(sy); sx = warp_sum(sx); cnt = warp_sum(cnt);
    if (lane == 0) { atomicAdd(&s_sum[0], sy); atomicAdd(&s_sum[1], sx); atomicAdd(&s_sum[2], cnt); }
    __syncthreads();
    if (tid == 0) {
        F.field_y = (double)s_sum[0] / (double)s_sum[2];
        F.field_x = (double)s_sum[1] / (double)s_sum[2];
    }
}

// ------------------------------------------------------------------------------------------------ BB finder
struct WlComp {
    int area[WL_MAXC];
    int y0[WL_MAXC], y1[WL_MAXC], x0[WL_MAXC], x1[WL_MAXC];
    int border[WL_MAXC];
    int root[WL_MAXC];
};

__global__ void __launch_bounds__(WL_THREADS)
k_wl_bb(const WlConst* __restrict__ cc, const uint16_t* __restrict__ base, const WlFrame* __restrict__ wf, double* __restrict__ samples,
        unsigned short* __restrict__ cid_all, WlComp* __restrict__ comp_all, epid_wl_result* __restrict__ res,
        epid_disk_result* __restrict__ dres, const uint16_t* const* __restrict__ item_src = nullptr,
        const epid_disk_params* __restrict__ item_loc = nullptr) {
    extern __shared__ __align__(16) unsigned char smraw[];
    __shared__ int s_i[16];
    __shared__ int s_added;
    __shared__ double s_d[8 + 2 * WL_WARPS];
    __shared__ double s_pts[2 * WL_MAXPTS];
    __shared__ int s_hist50[50];
    __shared__ int s_lvl[4 * (2 * WL_TILE + 2)];      // per half-row level: min / max of the doubled column coordinate
    const WlConst& c = *cc;
    const int fi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const WlFrame F = wf[fi];
    const bool loc = c.loc_mode != 0;
    // locator items (launch_disk_items): block = item, each with its own source frame and search parameters
    const epid_disk_params& L = item_loc ? item_loc[fi] : c.loc;
    epid_wl_result r_unused;
    epid_wl_result& R = loc ? r_unused : res[fi];      // the locator reports through dres
    if (loc && tid == 0) { dres[fi].status = F.status; dres[fi].n_points = 0; dres[fi].n_regions = 0; dres[fi].passes = 0; }
    if (tid == 0) {
        R.status = F.status;
        R.inverted = F.flip;
        R.crop_px = F.crop;
        R.height = F.h;
        R.width = F.w;
        R.n_bbs = 0;
        R.threshold_passes = 0;
    }
    if (F.status != EPID_WL_OK) return;
    const int H = c.H, W = c.W;
    const uint16_t* f = item_src ? item_src[fi] : base + (size_t)fi * H * W;
    const int h = F.h, w = F.w, crop = F.crop;
    const double dpmm = c.p.dpmm, Dd = (double)F.D;
    // ---- SizedDiskLocator.from_center_physical((0, 0), window 40 + bb) (metrics/image.py:564-612)
    const double bb_d = loc ? 2 * L.radius_mm : c.p.bb_size_mm;
    const double winx = loc ? L.window_w : (40 + bb_d) * dpmm, winy = loc ? L.window_h : (40 + bb_d) * dpmm;
    const double ex = loc ? L.expected_x : (double)w / 2, ey = loc ? L.expected_y : (double)h / 2;
    // metrics/image.py:583-591: floor / ceil bounds, the slice clips at the image edge
    const int left = min(max((int)floor(ex - winx / 2), 0), w), right = max(min((int)ceil(ex + winx / 2), w), 0);
    const int top = min(max((int)floor(ey - winy / 2), 0), h), bottom = max(min((int)ceil(ey + winy / 2), h), 0);
    const int wh = bottom - top, ww = right - left;
    if (loc && tid == 0) { dres[fi].left = left; dres[fi].top = top; }
    if (loc && (wh <= 0 || ww <= 0)) { if (tid == 0) dres[fi].status = EPID_WL_NO_BB; return; }      // empty sample
    if (wh < 3 || ww < 3 || wh > c.win_edge || ww > c.win_edge) {
        if (tid == 0) { R.status = EPID_WL_CAPACITY; if (loc) dres[fi].status = (wh < 3 || ww < 3) ? EPID_WL_NO_BB : EPID_WL_CAPACITY; }
        return;
    }
    const int npx = wh * ww;
    int* parent = reinterpret_cast<int*>(smraw);                         // npx ints (shared): union-find forest of the window
    unsigned short* cid = cid_all + (size_t)fi * WL_MAXWIN * WL_MAXWIN;  // component id of a root pixel (HBM scratch, L2 resident)
    WlComp* comp = comp_all + fi;                                        // per-component accumulators (HBM scratch)
    unsigned char* tile = reinterpret_cast<unsigned char*>(parent + c.win_edge * c.win_edge);   // WL_TILE^2: candidate mask / flood states
    unsigned char* tile2 = tile + WL_TILE * WL_TILE;                     // border image of the perimeter
    double* smp = samples + (size_t)fi * WL_MAXWIN * WL_MAXWIN;
    // ---- sample = stretch(invert(image[window])) with the reference's fp64 operation order
    uint32_t gmin = 0xffffffffu, gmax = 0;
    for (int i = tid; i < npx; i += WL_THREADS) {
        const int y = i / ww, x = i - y * ww;
        const uint32_t g = wl_T(F, f[(size_t)(top + y + crop) * W + (left + x + crop)]) - F.mn;
        gmin = min(gmin, g);
        gmax = max(gmax, g);
    }
    gmin = warp_min(gmin);
    gmax = warp_max(gmax);
    if (lane == 0) { s_i[wid] = (int)gmin; s_i[8 + wid] = (int)gmax; }
    __syncthreads();
    gmin = (uint32_t)s_i[0]; gmax = (uint32_t)s_i[8];
    for (int k = 1; k < WL_WARPS; k++) { gmin = min(gmin, (uint32_t)s_i[k]); gmax = max(gmax, (uint32_t)s_i[8 + k]); }
    __syncthreads();
    if (gmin == gmax) { if (tid == 0) { R.status = EPID_WL_NO_BB; if (loc) dres[fi].status = EPID_WL_NO_BB; } return; }     // stretch divides by zero, nothing is found
    const double amin = (double)gmin / Dd, amax = (double)gmax / Dd;
    const bool inv = loc ? (L.invert != 0) : !c.p.low_density_bb;
    // invert: b = -a + max + min (decreasing); stretch: (b - bmin) / (bmax - bmin) * 1, then ground with value 0
    const double bmin = inv ? (-amax + amax) + amin : amin, bmax = inv ? (-amin + amax) + amin : amax;
    const double cmax = bmax - bmin;
    for (int i = tid; i < npx; i += WL_THREADS) {
        const int y = i / ww, x = i - y * ww;
        const uint32_t g = wl_T(F, f[(size_t)(top + y + crop) * W + (left + x + crop)]) - F.mn;
        const double a = (double)g / Dd;
        const double b = inv ? (-a + amax) + amin : a;
        const double n_ = (b - bmin) / cmax;
        const double st = n_ * (double)(1 - 0);
        smp[i] = (st - 0.0) + 0.0;            // ground(stretched, value=0): the minimum of the stretched sample is exactly 0
    }
    __syncthreads();
    // ---- find_features (metrics/utils.py:66-190)
    const double radius_mm = bb_d / 2;
    // _calculate_bb_tolerance: np.interp(bb_diameter, (1.5, 30), (2, 4)) (winston_lutz.py:1062-1067)
    double tol;
    if (loc) tol = L.tolerance_mm;
    else if (bb_d <= 1.5) tol = 2.0;
    else if (bb_d >= 30.0) tol = 4.0;
    else { const double slope = (4.0 - 2.0) / (30.0 - 1.5); tol = slope * (bb_d - 1.5) + 2.0; }
    // detection conditions (metrics/features.py): all five for Winston-Lutz, the caller's subset for the stand-alone locator
    const int cm = loc ? L.conditions : 31;
    const bool c_size = cm & 1, c_round = cm & 2, c_circ = cm & 4, c_sym = cm & 8, c_solid = cm & 16, c_modest = cm & 32;
    const int max_number = loc ? min(max(L.max_number, 1), WL_MAXPTS) : 1;
    const double min_sep = loc ? L.min_separation_px : 5.0 * dpmm;      // deduplicate_points_and_boundaries (metrics/utils.py:14-37)
    const double PI = 3.141592653589793;
    const double larger_area = PI * ((radius_mm + tol) * (radius_mm + tol));
    const double smaller_area = fmax(PI * ((radius_mm - tol) * (radius_mm - tol)), 2.0);
    const double imin = 0.0, imax = 1.0;
    const double step = (imax - imin) / 50;
    double cutoff = imin + step;
    int npts = 0, passes = 0, fatal = 0, nreg = 0;
    while (cutoff <= imax && npts < max_number) {
        passes++;
        nreg = 0;                              // find_features returns the regions of the LAST threshold visited
        // -- measure.label(sample > cutoff, connectivity=1): union-find, roots = first pixel in raster order
        // Every pixel starts at the first pixel of its horizontal run (a warp per row: ballot + bit scan, carried across the 32-pixel
        // chunks), so only vertical merges remain, one per pair of overlapping runs (at the first pixel of the overlap); finds halve
        // their paths.  Roots are still the smallest index of a component.
        for (int y = wid; y < wh; y += WL_WARPS) {
            int carry = -1;                    // run start (column) of the run that reaches the end of the previous chunk
            for (int x0 = 0; x0 < ww; x0 += 32) {
                const int x = x0 + lane;
                const bool fg = x < ww && smp[y * ww + x] > cutoff;
                const unsigned bal = __ballot_sync(0xffffffffu, fg);
                int start = -1;
                if (fg) {
                    const unsigned zb = ~bal & ((1u << lane) - 1u);        // background pixels of the chunk to the left of this lane
                    start = zb ? x0 + (32 - __clz(zb)) : (carry >= 0 ? carry : x0);
                }
                if (x < ww) parent[y * ww + x] = fg ? y * ww + start : -1;
                carry = __shfl_sync(0xffffffffu, start, 31);
            }
        }
        __syncthreads();
        for (int i = tid; i < npx; i += WL_THREADS) {
            if (i < ww || parent[i] < 0 || parent[i - ww] < 0) continue;
            const int x = i % ww;
            if (x == 0 || parent[i - 1] < 0 || parent[i - ww - 1] < 0) gl_union(parent, i, i - ww);
        }
        __syncthreads();
        for (int i = tid; i < npx; i += WL_THREADS) if (parent[i] >= 0) parent[i] = gl_find(parent, i);
        __syncthreads();
        // -- component ids in label (raster) order: exclusive scan of the root flags
        if (tid == 0) s_i[0] = 0;
        __syncthreads();
        {
            int base_c = 0;
            for (int b0 = 0; b0 < npx; b0 += WL_THREADS) {
                const int i = b0 + tid;
                const bool isroot = i < npx && parent[i] == i;
                const unsigned bal = __ballot_sync(0xffffffffu, isroot);
                if (lane == 0) s_i[1 + wid] = __popc(bal);
                __syncthreads();
                int woff = 0, tot = 0;
                for (int k = 0; k < WL_WARPS; k++) { const int cnt = s_i[1 + k]; if (k < wid) woff += cnt; tot += cnt; }
                __syncthreads();
                if (isroot) {
                    const int id = base_c + woff + __popc(bal & ((1u << lane) - 1u));
                    cid[i] = (unsigned short)min(id, 0xffff);
                    if (id < WL_MAXC) { comp->area[id] = 0; comp->y0[id] = wh; comp->y1[id] = -1; comp->x0[id] = ww; comp->x1[id] = -1; comp->border[id] = 0; comp->root[id] = i; }
                }
                base_c += tot;
            }
            if (tid == 0) s_i[0] = base_c;
        }
        __syncthreads();
        const int ncomp_all = s_i[0];
        const int ncomp = min(ncomp_all, WL_MAXC);
        __syncthreads();
        if (ncomp_all > WL_MAXC) { fatal = 1; break; }
        // area / bounding box per component: the 32 raster-consecutive pixels of a warp mostly belong to one or two components, so the
        // warp combines its lanes per component id (match.any + redux) and issues one set of atomics per id instead of one per pixel
        for (int i0 = 0; i0 < npx; i0 += WL_THREADS) {
            const int i = i0 + tid;
            int id = -1, y = 0, x = 0;
            if (i < npx) {
                const int r = parent[i];
                if (r >= 0) {
                    id = cid[r];
                    if (id >= WL_MAXC) id = -1;
                    y = i / ww; x = i - y * ww;
                }
            }
            const unsigned act = __ballot_sync(0xffffffffu, id >= 0);
            if (id >= 0) {
                const unsigned peers = __match_any_sync(act, id);
                const int cnt = __popc(peers);
                const int ymin = __reduce_min_sync(peers, y), ymax = __reduce_max_sync(peers, y);
                const int xmin = __reduce_min_sync(peers, x), xmax = __reduce_max_sync(peers, x);
                if (lane == __ffs(peers) - 1) {
                    atomicAdd(&comp->area[id], cnt);
                    atomicMin(&comp->y0[id], ymin); atomicMax(&comp->y1[id], ymax);
                    atomicMin(&comp->x0[id], xmin); atomicMax(&comp->x1[id], xmax);
                    if (ymin == 0 || xmin == 0 || ymax == wh - 1 || xmax == ww - 1) comp->border[id] = 1;      // segmentation.clear_border
                }
            }
        }
        __syncthreads();
        // -- regions in label order through the detection conditions (metrics/features.py:7-68)
        for (int id = 0; id < ncomp; id++) {
            if (comp->border[id]) continue;
            const int by0 = comp->y0[id], by1 = comp->y1[id] + 1, bx0 = comp->x0[id], bx1 = comp->x1[id] + 1;
            const int bh = by1 - by0, bw = bx1 - bx0;
            const double bbox_area = (double)bh * (double)bw;
            // cheap necessary conditions of is_right_size_bb: area <= area_filled <= bbox area
            if (c_size && (!(smaller_area < bbox_area / (dpmm * dpmm)) || !((double)comp->area[id] / (dpmm * dpmm) < larger_area))) continue;
            if (bh + 2 > WL_TILE || bw + 2 > WL_TILE) {
                // a region this large cannot be round, symmetric and of the right size at once unless the tile is too small
                if (!c_size || !c_round || bbox_area * (PI / 4 * 0.8) / (dpmm * dpmm) < larger_area) fatal = 1;
                continue;
            }
            const int th = bh + 2, tw = bw + 2;
            const int root = comp->root[id];
            for (int i = tid; i < th * tw; i += WL_THREADS) {
                const int ty = i / tw, tx = i - ty * tw;
                const int y = by0 - 1 + ty, x = bx0 - 1 + tx;
                unsigned char m = 0;
                if (ty >= 1 && ty <= bh && tx >= 1 && tx <= bw) m = parent[y * ww + x] == root ? 1 : 0;
                tile[i] = m;
                tile2[i] = m;
            }
            __syncthreads();
            wl_flood_outside(tile, th, tw);
            int filled = 0;
            for (int i = tid; i < th * tw; i += WL_THREADS) filled += tile[i] != 2 ? 1 : 0;
            filled = warp_sum(filled);
            if (lane == 0) s_i[1 + wid] = filled;
            __syncthreads();
            filled = 0;
            for (int k = 0; k < WL_WARPS; k++) filled += s_i[1 + k];
            __syncthreads();
            // is_right_size_bb
            const double bb_area = (double)filled / (dpmm * dpmm);
            if (c_size && !(smaller_area < bb_area && bb_area < larger_area)) continue;
            // is_modest_size (winston_lutz.py:598-606); find_features hands it the RADIUS as bb_size (metrics/utils.py:144-150)
            if (c_modest && !(fmax(PI * (((radius_mm - 2) / 2) * ((radius_mm - 2) / 2)), 2.0) < bb_area &&
                              bb_area < PI * (((radius_mm + 2) / 2) * ((radius_mm + 2) / 2)))) continue;
            // is_round
            const double ratio = (double)filled / bbox_area;
            if (c_round && !(PI / 4 * 1.2 > ratio && ratio > PI / 4 * 0.8)) continue;
            // is_right_circumference: skimage.measure.perimeter(image, neighborhood=4) on the region mask (tile2 = mask)
            if (tid < 50) s_hist50[tid] = 0;
            __syncthreads();
            for (int i = tid; i < th * tw; i += WL_THREADS) {
                const int ty = i / tw, tx = i - ty * tw;
                unsigned char b = 0;
                if (tile2[i] == 1) {
                    // eroded = centre and its 4 neighbours inside the mask (border_value 0); the margin guarantees neighbours exist
                    const bool er = tile2[i - 1] == 1 && tile2[i + 1] == 1 && tile2[i - tw] == 1 && tile2[i + tw] == 1;
                    b = er ? 0 : 1;
                }
                tile[i] = b;      // border image
                (void)ty; (void)tx;
            }
            __syncthreads();
            for (int i = tid; i < th * tw; i += WL_THREADS) {
                const int ty = i / tw, tx = i - ty * tw;
                int v = 0;
                for (int dy = -1; dy <= 1; dy++)
                    for (int dx = -1; dx <= 1; dx++) {
                        const int yy = ty + dy, xx = tx + dx;
                        if (yy < 0 || yy >= th || xx < 0 || xx >= tw) continue;
                        if (tile[yy * tw + xx]) v += (dy == 0 && dx == 0) ? 1 : ((dy == 0 || dx == 0) ? 2 : 10);
                    }
                if (v > 0 && v < 50) atomicAdd(&s_hist50[v], 1);
            }
            __syncthreads();
            double perim = 0.0;
            {
                const double w1 = 1.0, w2 = sqrt(2.0), w3 = (1 + sqrt(2.0)) / 2;
                for (int k = 0; k < 50; k++) {
                    double wk = 0.0;
                    if (k == 5 || k == 7 || k == 15 || k == 17 || k == 25 || k == 27) wk = w1;
                    else if (k == 21 || k == 33) wk = w2;
                    else if (k == 13 || k == 23) wk = w3;
                    perim += (double)s_hist50[k] * wk;
                }
            }
            __syncthreads();
            const double per_mm = perim / dpmm;
            if (c_circ && !(2 * PI * (radius_mm + tol) > per_mm && per_mm > 2 * PI * (radius_mm - tol))) continue;
            // is_symmetric
            {
                const double y = (double)bh, x = (double)bw;
                if (c_sym && (x > fmax(y * 1.05, y + 3) || x < fmin(y * 0.95, y - 3))) continue;
            }
            // is_solid: area / area_convex > 0.9; convex hull of the pixels' diamond offsets (r +- 0.5, c), (r, c +- 0.5).
            // Per half-row level L = 2 r + {-1, 0, 1} keep the extreme doubled column coordinates; the hull's column extent at an
            // integer row is the extreme interpolation between any two levels that bracket it.
            const int nlev = 2 * bh + 1;          // levels -1 .. 2 bh - 1  (index = L + 1)
            for (int i = tid; i < nlev; i += WL_THREADS) { s_lvl[2 * i] = 0x7fffffff; s_lvl[2 * i + 1] = -0x7fffffff; }
            __syncthreads();
            for (int i = tid; i < bh * bw; i += WL_THREADS) {
                const int r = i / bw, cidx = i - r * bw;
                if (tile2[(r + 1) * tw + (cidx + 1)] != 1) continue;
                // doubled coordinates: (2r, 2c +- 1) on level 2r; (2r +- 1, 2c) on levels 2r +- 1
                atomicMin(&s_lvl[2 * (2 * r + 1)], 2 * cidx - 1); atomicMax(&s_lvl[2 * (2 * r + 1) + 1], 2 * cidx + 1);
                atomicMin(&s_lvl[2 * (2 * r)], 2 * cidx); atomicMax(&s_lvl[2 * (2 * r) + 1], 2 * cidx);
                atomicMin(&s_lvl[2 * (2 * r + 2)], 2 * cidx); atomicMax(&s_lvl[2 * (2 * r + 2) + 1], 2 * cidx);
            }
            __syncthreads();
            int convex = 0;
            for (int r = tid; r < bh; r += WL_THREADS) {
                // column extent (doubled coordinates) of the hull at level Lr = 2 r (index 2 r + 1)
                const int li = 2 * r + 1;
                double xl = (double)s_lvl[2 * li], xr = (double)s_lvl[2 * li + 1];
                for (int a = 0; a < li; a++) {
                    if (s_lvl[2 * a + 1] == -0x7fffffff) continue;
                    for (int b = li + 1; b < nlev; b++) {
                        if (s_lvl[2 * b + 1] == -0x7fffffff) continue;
                        const double t = (double)(li - a) / (double)(b - a);
                        const double l = (double)s_lvl[2 * a] + t * (double)(s_lvl[2 * b] - s_lvl[2 * a]);
                        const double rr = (double)s_lvl[2 * a + 1] + t * (double)(s_lvl[2 * b + 1] - s_lvl[2 * a + 1]);
                        xl = fmin(xl, l);
                        xr = fmax(xr, rr);
                    }
                }
                // pixel centres (doubled column 2 c) with xl - eps <= 2 c <= xr + eps
                const int c_lo = (int)ceil((xl - 2e-10) / 2), c_hi = (int)floor((xr + 2e-10) / 2);
                if (c_hi >= c_lo) convex += c_hi - c_lo + 1;
            }
            convex = warp_sum(convex);
            if (lane == 0) s_i[1 + wid] = convex;
            __syncthreads();
            convex = 0;
            for (int k = 0; k < WL_WARPS; k++) convex += s_i[1 + k];
            __syncthreads();
            if (c_solid && !((double)comp->area[id] / (double)convex > 0.9)) continue;
            // -- accepted: centroid_weighted (local moments of the stretched sample over the region, + bbox origin)
            if (tid < 4) s_lvl[tid] = 0;      // (the hull levels are no longer needed) 64-bit accumulators of the unweighted moments
            __syncthreads();
            double sw = 0, swr = 0, swc = 0;
            unsigned long long sr_i = 0, sc_i = 0;      // unweighted first moments (regionprops.centroid)
            for (int i = tid; i < bh * bw; i += WL_THREADS) {
                const int r = i / bw, cidx = i - r * bw;
                if (tile2[(r + 1) * tw + (cidx + 1)] != 1) continue;
                const double wv = smp[(by0 + r) * ww + (bx0 + cidx)];
                sw += wv;
                swr += (double)r * wv;
                swc += (double)cidx * wv;
                sr_i += (unsigned long long)r;
                sc_i += (unsigned long long)cidx;
            }
            sr_i = warp_sum(sr_i); sc_i = warp_sum(sc_i);
            if (loc && lane == 0) { atomicAdd(reinterpret_cast<unsigned long long*>(&s_lvl[0]), sr_i); atomicAdd(reinterpret_cast<unsigned long long*>(&s_lvl[2]), sc_i); }
            sw = warp_sum(sw); swr = warp_sum(swr); swc = warp_sum(swc);
            if (lane == 0) { s_d[8 + wid] = sw; s_d[8 + WL_WARPS + wid] = swr; }
            __syncthreads();
            double tw_ = 0, tr_ = 0;
            for (int k = 0; k < WL_WARPS; k++) { tw_ += s_d[8 + k]; tr_ += s_d[8 + WL_WARPS + k]; }
            __syncthreads();
            if (lane == 0) s_d[8 + wid] = swc;
            __syncthreads();
            double tc_ = 0;
            for (int k = 0; k < WL_WARPS; k++) tc_ += s_d[8 + k];
            __syncthreads();
            if (tid == 0) {
                const double px = tc_ / tw_ + (double)bx0;       // Point(x = weighted_centroid[1], y = weighted_centroid[0])
                const double py = tr_ / tw_ + (double)by0;
                bool keep = npts < WL_MAXPTS;
                for (int k = 0; k < npts && keep; k++) {
                    const double dx = px - s_pts[2 * k], dy = py - s_pts[2 * k + 1];
                    if (sqrt(dx * dx + dy * dy + 0.0) < min_sep) keep = false;
                }
                if (keep) { s_pts[2 * npts] = px; s_pts[2 * npts + 1] = py; }
                s_added = keep ? 1 : 0;
                if (loc && nreg < EPID_DISK_MAX) {
                    epid_disk_result& D = dres[fi];
                    const double area = (double)comp->area[id];
                    D.r_area[nreg] = area;
                    D.r_filled_area[nreg] = (double)filled;
                    D.r_perimeter[nreg] = perim;
                    D.r_convex_area[nreg] = (double)convex;
                    D.r_bbox[nreg][0] = by0; D.r_bbox[nreg][1] = bx0; D.r_bbox[nreg][2] = by1; D.r_bbox[nreg][3] = bx1;
                    D.r_centroid_y[nreg] = (double)*reinterpret_cast<unsigned long long*>(&s_lvl[0]) / area + (double)by0;
                    D.r_centroid_x[nreg] = (double)*reinterpret_cast<unsigned long long*>(&s_lvl[2]) / area + (double)bx0;
                    D.r_wcentroid_y[nreg] = py;
                    D.r_wcentroid_x[nreg] = px;
                }
            }
            nreg++;
            __syncthreads();
            npts += s_added;
            __syncthreads();
        }
        if (fatal) break;
        cutoff += step;
    }
    if (loc) {      // stand-alone locator: points in image coordinates + the regions of the last threshold
        if (tid == 0) {
            epid_disk_result& D = dres[fi];
            D.passes = passes;
            D.status = fatal ? EPID_WL_CAPACITY : EPID_WL_OK;
            D.n_points = npts;
            D.n_regions = min(nreg, EPID_DISK_MAX);
            for (int k = 0; k < npts; k++) { D.x[k] = s_pts[2 * k] + (double)left; D.y[k] = s_pts[2 * k + 1] + (double)top; }
        }
        return;
    }
    // ---- matching and results (thread 0)
    if (tid == 0) {
        R.threshold_passes = passes;
        if (fatal) { R.status = EPID_WL_CAPACITY; return; }
        if (npts < 1) { R.status = EPID_WL_NO_BB; return; }
        R.n_bbs = npts;
        const double epx = (double)w / 2 - 0.5, epy = (double)h / 2 - 0.5;      // image.center / cax (core/image.py:526-533, 1550-1580)
        // find_bb_matches (winston_lutz.py:808-829): nearest detected point to the nominal position (ISO: the EPID centre)
        double best = 0;
        int bi = -1;
        for (int k = 0; k < npts; k++) {
            const double px = s_pts[2 * k] + (double)left, py = s_pts[2 * k + 1] + (double)top;
            s_pts[2 * k] = px;
            s_pts[2 * k + 1] = py;
            const double dx = epx - px, dy = epy - py;
            const double d = sqrt(dx * dx + dy * dy + 0.0);
            if (bi < 0 || d < best) { best = d; bi = k; }
        }
        const bool bb_ok = best < c.p.bb_proximity_mm * dpmm;
        const double fdx = epx - F.field_x, fdy = epy - F.field_y;
        const bool field_ok = sqrt(fdx * fdx + fdy * fdy + 0.0) < c.p.bb_proximity_mm * dpmm;
        if (bb_ok != field_ok) { R.status = EPID_WL_MISMATCH; return; }
        if (!field_ok) { R.status = EPID_WL_NO_FIELD; return; }
        R.bb_x = s_pts[2 * bi];
        R.bb_y = s_pts[2 * bi + 1];
        R.field_x = F.field_x;
        R.field_y = F.field_y;
        R.epid_x = epx;
        R.epid_y = epy;
        // cax2bb_vector / distance, cax2epid_vector / distance (winston_lutz.py:1186-1209)
        R.cax2bb_x = (R.bb_x - R.field_x) / dpmm;
        R.cax2bb_y = (R.bb_y - R.field_y) / dpmm;
        {
            const double dx = R.field_x - R.bb_x, dy = R.field_y - R.bb_y;
            R.cax2bb_distance = sqrt(dx * dx + dy * dy + 0.0) / dpmm;
        }
        R.cax2epid_x = (epx - R.field_x) / dpmm;
        R.cax2epid_y = (epy - R.field_y) / dpmm;
        {
            const double dx = R.field_x - epx, dy = R.field_y - epy;
            R.cax2epid_distance = sqrt(dx * dx + dy * dy + 0.0) / dpmm;
        }
    }
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_wl2d_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_wl_params* p, epid_wl_result* results) {
    EPID_REQUIRE(ctx && frames && p && results, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(frames->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "Winston-Lutz frames must be uint16");
    EPID_REQUIRE(p->dpmm > 0 && p->bb_size_mm > 0, EPID_ERR_INVALID, "dpmm and bb_size_mm must be positive");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = frames->n, H = frames->h, W = frames->w;
    EPID_REQUIRE(H >= 16 && W >= 16, EPID_ERR_UNSUPPORTED, "frame too small");
    WlConst hc;
    memset(&hc, 0, sizeof(hc));
    hc.p = *p;
    hc.H = H;
    hc.W = W;
    hc.field_tile_cap = 200 * 1024;
    const int chunk = n < 512 ? n : 512;       // 256 KB of histogram + 400 KB of sample per frame in flight
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    const size_t o_cst = sz(sizeof(WlConst)), o_fr = sz(sizeof(WlFrame) * chunk), o_res = sz(sizeof(epid_wl_result) * chunk);
    const size_t o_hist = sz(sizeof(uint32_t) * (size_t)chunk * 65536), o_smp = sz(sizeof(double) * (size_t)chunk * WL_MAXWIN * WL_MAXWIN);
    const size_t o_cid = sz(sizeof(unsigned short) * (size_t)chunk * WL_MAXWIN * WL_MAXWIN), o_cmp = sz(sizeof(WlComp) * (size_t)chunk);
    int rc = ensure_scratch(ctx, o);
    if (rc != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    cudaStream_t st = ctx->stream;
    // the BB window is (40 + bb) mm: size the shared-memory forest for it, not for the largest window the kernel supports
    int win_edge = (int)ceil((40 + p->bb_size_mm) * p->dpmm) + 2;
    if (win_edge > WL_MAXWIN) win_edge = WL_MAXWIN;      // larger windows report EPID_WL_CAPACITY per frame
    if (win_edge < 8) win_edge = 8;
    hc.win_edge = win_edge;
    const size_t bb_smem = sizeof(int) * (size_t)win_edge * win_edge + 2 * WL_TILE * WL_TILE + 64;
    const size_t bb_smem_max = sizeof(int) * WL_MAXWIN * WL_MAXWIN + 2 * WL_TILE * WL_TILE + 64;
    EPID_CUDA(cudaMemcpyAsync(base + o_cst, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    EPID_SMEM_OPT_IN(ctx, k_wl_field, (size_t)hc.field_tile_cap);
    EPID_SMEM_OPT_IN(ctx, k_wl_bb, bb_smem_max);
    for (int c0 = 0; c0 < n; c0 += chunk) {
        const int cn = n - c0 < chunk ? n - c0 : chunk;
        const uint16_t* d_frames = (const uint16_t*)frames->dptr + (size_t)c0 * H * W;
        EPID_CUDA(cudaMemsetAsync(base + o_hist, 0, sizeof(uint32_t) * (size_t)cn * 65536, st));
        EPID_CUDA(cudaMemsetAsync(base + o_res, 0, sizeof(epid_wl_result) * cn, st));
        k_wl_hist<<<dim3(WL_HPARTS, cn), 256, 0, st>>>(d_frames, H, W, (uint32_t*)(base + o_hist));
        k_wl_front<<<cn, WL_THREADS, 0, st>>>((const WlConst*)(base + o_cst), d_frames, (uint32_t*)(base + o_hist), (WlFrame*)(base + o_fr));
        k_wl_bbox<<<dim3(WL_BBOX_PARTS, cn), WL_THREADS, 0, st>>>((const WlConst*)(base + o_cst), d_frames, (WlFrame*)(base + o_fr));
        k_wl_field<<<cn, WL_THREADS, hc.field_tile_cap, st>>>((const WlConst*)(base + o_cst), d_frames, (WlFrame*)(base + o_fr));
        k_wl_bb<<<cn, WL_THREADS, bb_smem, st>>>((const WlConst*)(base + o_cst), d_frames, (const WlFrame*)(base + o_fr), (double*)(base + o_smp),
                                                 (unsigned short*)(base + o_cid), (WlComp*)(base + o_cmp), (epid_wl_result*)(base + o_res), nullptr);
        ctx->launches += 5;
        EPID_CUDA(cudaGetLastError());
        EPID_CUDA(cudaMemcpyAsync(results + c0, base + o_res, sizeof(epid_wl_result) * cn, cudaMemcpyDeviceToHost, st));
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("Winston-Lutz pipeline failed: %s", cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    }
    return EPID_OK;
}

namespace epid {
__global__ void k_loc_init(WlFrame* wf, int n, int H, int W) {
    // identity pixel map: the locator's sample is stretch(invert(image[window])) of the RAW frame (metrics/image.py:592-596)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    WlFrame f;
    memset(&f, 0, sizeof(f));
    f.status = EPID_WL_OK;
    f.h = H; f.w = W;
    f.mn = 0; f.D = 1;
    wf[i] = f;
}
}  // namespace epid

namespace epid {
__global__ void k_loc_items_init(const WlItemMap* __restrict__ maps, WlFrame* wf, int n, int H, int W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    WlFrame f;
    memset(&f, 0, sizeof(f));
    f.status = maps[i].status;
    f.h = H; f.w = W;
    f.mn = maps[i].mn; f.D = maps[i].D;
    wf[i] = f;
}

static size_t disk_items_layout(int n, size_t* o_cst, size_t* o_fr, size_t* o_smp, size_t* o_cid, size_t* o_cmp) {
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    *o_cst = sz(sizeof(WlConst)); *o_fr = sz(sizeof(WlFrame) * n);
    *o_smp = sz(sizeof(double) * (size_t)n * WL_MAXWIN * WL_MAXWIN);
    *o_cid = sz(sizeof(unsigned short) * (size_t)n * WL_MAXWIN * WL_MAXWIN); *o_cmp = sz(sizeof(WlComp) * (size_t)n);
    return o;
}

size_t disk_items_scratch_bytes(int n_items) {
    size_t a, b, c, d, e;
    return disk_items_layout(n_items, &a, &b, &c, &d, &e);
}

int launch_disk_items(epid_ctx* ctx, cudaStream_t st, void* scratch, int n, int H, int W, double dpmm, double max_window_px,
                      const uint16_t* const* d_src, const WlItemMap* d_maps, const epid_disk_params* d_loc, epid_disk_result* d_res) {
    size_t o_cst, o_fr, o_smp, o_cid, o_cmp;
    disk_items_layout(n, &o_cst, &o_fr, &o_smp, &o_cid, &o_cmp);
    char* base = (char*)scratch;
    WlConst hc;
    memset(&hc, 0, sizeof(hc));
    hc.p.dpmm = dpmm;
    hc.H = H;
    hc.W = W;
    hc.loc_mode = 1;
    int win_edge = (int)ceil(max_window_px) + 2;
    if (win_edge > WL_MAXWIN) win_edge = WL_MAXWIN;      // larger windows report EPID_WL_CAPACITY per item
    if (win_edge < 8) win_edge = 8;
    hc.win_edge = win_edge;
    const size_t bb_smem = sizeof(int) * (size_t)win_edge * win_edge + 2 * WL_TILE * WL_TILE + 64;
    EPID_CUDA(cudaMemcpyAsync(base + o_cst, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    EPID_SMEM_OPT_IN(ctx, k_wl_bb, sizeof(int) * WL_MAXWIN * WL_MAXWIN + 2 * WL_TILE * WL_TILE + 64);
    k_loc_items_init<<<(n + 127) / 128, 128, 0, st>>>(d_maps, (WlFrame*)(base + o_fr), n, H, W);
    k_wl_bb<<<n, WL_THREADS, bb_smem, st>>>((const WlConst*)(base + o_cst), nullptr, (const WlFrame*)(base + o_fr), (double*)(base + o_smp),
                                           (unsigned short*)(base + o_cid), (WlComp*)(base + o_cmp), nullptr, d_res, d_src, d_loc);
    ctx->launches += 2;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}
}  // namespace epid

extern "C" int32_t epid_disk_locate(epid_ctx* ctx, const epid_batch* frames, const epid_disk_params* p, epid_disk_result* results) {
    EPID_REQUIRE(ctx && frames && p && results, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(frames->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "disk locator frames must be uint16");
    EPID_REQUIRE(p->dpmm > 0 && p->radius_mm > 0 && p->window_w > 0 && p->window_h > 0, EPID_ERR_INVALID, "dpmm, radius and window must be positive");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = frames->n, H = frames->h, W = frames->w;
    WlConst hc;
    memset(&hc, 0, sizeof(hc));
    hc.p.dpmm = p->dpmm;
    hc.p.bb_size_mm = 2 * p->radius_mm;
    hc.H = H;
    hc.W = W;
    hc.loc_mode = 1;
    hc.loc = *p;
    int win_edge = (int)ceil(p->window_w > p->window_h ? p->window_w : p->window_h) + 2;
    if (win_edge > WL_MAXWIN) win_edge = WL_MAXWIN;      // larger windows report EPID_WL_CAPACITY per frame
    if (win_edge < 8) win_edge = 8;
    hc.win_edge = win_edge;
    const int chunk = n < 256 ? n : 256;
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    const size_t o_cst = sz(sizeof(WlConst)), o_fr = sz(sizeof(WlFrame) * chunk), o_res = sz(sizeof(epid_disk_result) * chunk);
    const size_t o_smp = sz(sizeof(double) * (size_t)chunk * WL_MAXWIN * WL_MAXWIN);
    const size_t o_cid = sz(sizeof(unsigned short) * (size_t)chunk * WL_MAXWIN * WL_MAXWIN), o_cmp = sz(sizeof(WlComp) * (size_t)chunk);
    int rc = ensure_scratch(ctx, o);
    if (rc != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    cudaStream_t st = ctx->stream;
    const size_t bb_smem = sizeof(int) * (size_t)win_edge * win_edge + 2 * WL_TILE * WL_TILE + 64;
    EPID_CUDA(cudaMemcpyAsync(base + o_cst, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    EPID_SMEM_OPT_IN(ctx, k_wl_bb, sizeof(int) * WL_MAXWIN * WL_MAXWIN + 2 * WL_TILE * WL_TILE + 64);
    for (int c0 = 0; c0 < n; c0 += chunk) {
        const int cn = n - c0 < chunk ? n - c0 : chunk;
        const uint16_t* d_frames = (const uint16_t*)frames->dptr + (size_t)c0 * H * W;
        EPID_CUDA(cudaMemsetAsync(base + o_res, 0, sizeof(epid_disk_result) * cn, st));
        k_loc_init<<<(cn + 127) / 128, 128, 0, st>>>((WlFrame*)(base + o_fr), cn, H, W);
        k_wl_bb<<<cn, WL_THREADS, bb_smem, st>>>((const WlConst*)(base + o_cst), d_frames, (const WlFrame*)(base + o_fr), (double*)(base + o_smp),
                                                 (unsigned short*)(base + o_cid), (WlComp*)(base + o_cmp), nullptr, (epid_disk_result*)(base + o_res));
        ctx->launches += 2;
        EPID_CUDA(cudaGetLastError());
        EPID_CUDA(cudaMemcpyAsync(results + c0, base + o_res, sizeof(epid_disk_result) * cn, cudaMemcpyDeviceToHost, st));
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("disk locator failed: %s", cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    }
    return EPID_OK;
}
