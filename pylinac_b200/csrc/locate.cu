// Whole-frame feature finders: GlobalSizedDiskLocator / GlobalSizedFieldLocator / GlobalFieldLocator (metrics/image.py:275-354,
// 727-956) and the threshold sweep they share with find_features (metrics/utils.py:66-190).
//
// The reference binarises the frame at up to 50 rising thresholds and runs skimage label / clear_border / regionprops on every one.
// Here every threshold is six launches over the WHOLE batch (frames never leave HBM, no host round trip inside the sweep):
//   k_gl_minmax      min / max of every frame (once)
//   k_gl_plan        the reference's fp64 cutoff sequence, converted into exact integer pixel thresholds: the sample a pixel stands
//                    for (invert / stretch / normalise in the reference's operation order) is monotone in the raw pixel value, so
//                    `sample > cutoff` is a threshold on the integer; found by bisection on that exact fp64 expression (once)
//   k_gl_init        parent[i] = i for foreground pixels (-1 otherwise)
//   k_ccl_union      ccl.cuh's union-find merge with the earlier neighbours (4- or 8-connectivity), roots = first pixel in raster
//                    order = skimage's label order
//   k_gl_flatten     parent[i] = root; root pixels reset their accumulators
//   k_gl_props       area / bounding box per region, warp-aggregated atomics on root-indexed arrays
//   k_gl_select      root pixels that survive clear_border and the cheap necessary conditions (area <= area_filled <= bbox area)
//                    become candidates
//   k_gl_analyze     CTA per candidate: region mask in a shared-memory tile (global scratch for regions beyond the tile), flood of
//                    the outside (binary_fill_holes), skimage perimeter (4-neighbourhood border, weighted 3 x 3 histogram), centroid /
//                    weighted centroid / equivalent diameter, the detection conditions -> accepted-region records
// The host merges the per-threshold records in the reference's order (threshold, then label) with its de-duplication and stop rule.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "ccl.cuh"

namespace epid {

constexpr int GL_THREADS = 256;
constexpr int GL_MAXTHR = 64;
constexpr int GL_CHUNK = 32;            // frames labelled at a time (scratch: 24 B per pixel and frame)
constexpr int GL_MAXCAND = 2048;          // candidates per frame and threshold
constexpr int GL_TILE_BYTES = 200 * 1024; // large shared-memory tile of the per-candidate analysis (regions up to ~450 x 450)
constexpr int GL_SMALL_TILE = 40 * 1024;  // small tile: the common case (regions up to ~200 x 200), several CTAs per SM

struct GlFrame {
    unsigned int mn, mx;
    int nthr;
    int dir[GL_MAXTHR];            // +1: foreground = raw >= T, -1: foreground = raw <= T
    unsigned int T[GL_MAXTHR];
    double cutoff[GL_MAXTHR];
};

struct GlCand { int root, x0, y0, x1, y1, area; };

__global__ void k_gl_minmax_init(GlFrame* gf, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { gf[i].mn = 0xffffffffu; gf[i].mx = 0; }
}

__global__ void k_gl_minmax(const uint16_t* __restrict__ frames, size_t per, GlFrame* gf) {
    const int f = blockIdx.y;
    const uint16_t* img = frames + (size_t)f * per;
    unsigned int mn = 0xffffu, mx = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (size_t)gridDim.x * blockDim.x) {
        const unsigned int v = img[i];
        mn = min(mn, v); mx = max(mx, v);
    }
    mn = warp_min(mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { atomicMin(&gf[f].mn, mn); atomicMax(&gf[f].mx, mx); }
}

// the fp64 sample the reference thresholds, as a function of the raw pixel value v of a frame with minimum mn and range D
//   mode 0 (find_features): stretch(invert?(array));  mode 1 (field locator): the array itself
//   kind 0: the array is the integer frame;  kind 1: the array is the ground()-ed and normalize()-d float image fl((v - mn) / D)
__device__ inline double gl_sample(int mode, int kind, int invert, unsigned int v, unsigned int mn, unsigned int D) {
    const double g = (double)(v - mn), Dd = (double)D;
    if (kind == 0) {
        if (mode == 1) return (double)v;
        const double gi = invert ? (double)(D - (v - mn)) : g;      // uint16 invert + ground: exact integers
        return ((gi / Dd) * 1.0 - 0.0) + 0.0;                       // normalize, * (max - min), ground(value=0) of the stretch
    }
    const double a = g / Dd;                                         // the float image
    if (mode == 1 || !invert) return mode == 1 ? a : ((a - 0.0) / 1.0 * 1.0 - 0.0) + 0.0;
    const double b = (-a + 1.0) + 0.0;                               // invert: -a + max + min
    return ((b - 0.0) / 1.0 * 1.0 - 0.0) + 0.0;
}

__global__ void k_gl_plan(GlFrame* gf, int n, int mode, int kind, int invert) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    GlFrame& F = gf[f];
    const unsigned int mn = F.mn, mx = F.mx, D = mx - mn;
    F.nthr = 0;
    if (D == 0) return;      // flat frame: stretch divides by zero / the sweep never enters its loop
    double imin, imax;
    if (mode == 0) { imin = 0.0; imax = 1.0; }
    else if (kind == 0) { imin = (double)mn; imax = (double)mx; }
    else { imin = 0.0; imax = 1.0; }
    const double spread = imax - imin, step = spread / 50;
    double cutoff = mode == 0 ? imin + step : imin + step * 5;
    const bool decreasing = mode == 0 && invert;
    int k = 0;
    while (cutoff <= imax && k < GL_MAXTHR) {
        // foreground(v) = sample(v) > cutoff, monotone in v: bisection for the boundary
        unsigned int lo = mn, hi = mx;      // increasing: smallest v with fg;  decreasing: largest v with fg
        int dir;
        unsigned int T;
        if (!decreasing) {
            dir = 1;
            if (!(gl_sample(mode, kind, invert, mx, mn, D) > cutoff)) T = mx + 1;      // nothing is foreground
            else {
                while (lo < hi) { const unsigned int mid = lo + (hi - lo) / 2; if (gl_sample(mode, kind, invert, mid, mn, D) > cutoff) hi = mid; else lo = mid + 1; }
                T = lo;
            }
        } else {
            dir = -1;
            if (!(gl_sample(mode, kind, invert, mn, mn, D) > cutoff)) { T = 0; dir = -2; }      // nothing is foreground
            else {
                while (lo < hi) { const unsigned int mid = lo + (hi - lo + 1) / 2; if (gl_sample(mode, kind, invert, mid, mn, D) > cutoff) lo = mid; else hi = mid - 1; }
                T = lo;
            }
        }
        F.dir[k] = dir; F.T[k] = T; F.cutoff[k] = cutoff;
        k++;
        cutoff += step;
    }
    F.nthr = k;
}

__device__ __forceinline__ bool gl_fg(const GlFrame& F, int k, unsigned int v) {
    const int d = F.dir[k];
    return d == 1 ? v >= F.T[k] : (d == -1 ? v <= F.T[k] : false);
}

// ------------------------------------------------------------------------------------------------ labelling
__global__ void k_gl_init(const uint16_t* __restrict__ frames, int HW, const GlFrame* __restrict__ gf, int k, int* __restrict__ parent,
                          int* __restrict__ ncand) {
    const int f = blockIdx.y;
    const GlFrame& F = gf[f];
    if (blockIdx.x == 0 && threadIdx.x == 0) ncand[f] = 0;
    const uint16_t* img = frames + (size_t)f * HW;
    int* par = parent + (size_t)f * HW;
    const bool live = k < F.nthr;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) par[i] = live && gl_fg(F, k, img[i]) ? i : -1;
}

__global__ void k_gl_flatten(int HW, int W, int H, int* __restrict__ parent, unsigned int* __restrict__ area, unsigned int* __restrict__ bx0,
                             unsigned int* __restrict__ bx1, unsigned int* __restrict__ by0, unsigned int* __restrict__ by1) {
    const int f = blockIdx.y;
    const size_t o = (size_t)f * HW;
    int* par = parent + o;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        if (par[i] < 0) continue;
        const int r = ccl_root(par, i);
        if (r == i) { area[o + i] = 0; bx0[o + i] = W; bx1[o + i] = 0; by0[o + i] = H; by1[o + i] = 0; }
        else par[i] = r;
    }
}

__global__ void k_gl_props(int HW, int W, const int* __restrict__ parent, unsigned int* __restrict__ area, unsigned int* __restrict__ bx0,
                           unsigned int* __restrict__ bx1, unsigned int* __restrict__ by0, unsigned int* __restrict__ by1) {
    const int f = blockIdx.y;
    const size_t o = (size_t)f * HW;
    const int* par = parent + o;
    const int lane = threadIdx.x & 31;
    // every warp walks 32 consecutive pixels: lanes with the same root are merged before the area / row atomics; the column
    // extremes are posted by the ends of every horizontal run only
    const int n32 = (HW + 31) / 32 * 32;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n32; i += gridDim.x * blockDim.x) {
        const int r = i < HW ? par[i] : -1;
        const unsigned int act = __ballot_sync(0xffffffffu, r >= 0);
        if (r < 0) continue;
        const unsigned int peers = __match_any_sync(act, r);
        const int first = __ffs(peers) - 1, last = 31 - __clz(peers);
        const int y = i / W, x = i - y * W;
        const int yf = __shfl_sync(peers, y, first), yl = __shfl_sync(peers, y, last);      // raster order: first / last row of the group
        if (lane == first) {
            atomicAdd(&area[o + r], (unsigned int)__popc(peers));
            atomicMin(&by0[o + r], (unsigned int)yf);
            atomicMax(&by1[o + r], (unsigned int)yl);
        }
        if (x == 0 || par[i - 1] < 0) atomicMin(&bx0[o + r], (unsigned int)x);
        if (x == W - 1 || par[i + 1] < 0) atomicMax(&bx1[o + r], (unsigned int)x);
    }
}

struct GlCfg {
    int mode, kind, invert, conn8, border;      // border: clear_border removes regions with a pixel in the outer `border` rows / columns
    int conditions;
    int H, W;
    double dpmm;
    double radius_mm, tol_mm;                    // disk conditions (bb_size = radius, tolerance)
    double field_w_mm, field_h_mm, field_tol_mm; // field conditions
    double bb_size_mm, rad_size_mm;              // is_modest_size / is_right_square_size
};

// condition bits (pylinac_b200/metrics/features.py)
constexpr int C_SIZE_BB = 1, C_ROUND = 2, C_CIRC = 4, C_SYM = 8, C_SOLID = 16, C_MODEST = 32, C_SQUARE = 64, C_SQ_SIZE = 128,
              C_SQ_PERIM = 256, C_AREA_SQ = 512;

__device__ inline void gl_area_bounds(const GlCfg& c, double* lo, double* hi) {
    // the intersection of the size windows of the requested conditions on area_filled / dpmm^2
    const double PI = 3.141592653589793;
    double l = -1e300, h = 1e300;
    if (c.conditions & C_SIZE_BB) {
        h = fmin(h, PI * ((c.radius_mm + c.tol_mm) * (c.radius_mm + c.tol_mm)));
        l = fmax(l, fmax(PI * ((c.radius_mm - c.tol_mm) * (c.radius_mm - c.tol_mm)), 2.0));
    }
    if (c.conditions & C_MODEST) {
        h = fmin(h, PI * (((c.bb_size_mm + 2) / 2) * ((c.bb_size_mm + 2) / 2)));
        l = fmax(l, fmax(PI * (((c.bb_size_mm - 2) / 2) * ((c.bb_size_mm - 2) / 2)), 2.0));
    }
    if (c.conditions & C_SQ_SIZE) {
        const double rs = fmax(c.rad_size_mm, 5.0);
        h = fmin(h, (rs + 5) * (rs + 5));
        l = fmax(l, (rs - 5) * (rs - 5));
    }
    if (c.conditions & C_AREA_SQ) {
        h = fmin(h, (c.field_w_mm + c.field_tol_mm) * (c.field_h_mm + c.field_tol_mm));
        l = fmax(l, (c.field_w_mm - c.field_tol_mm) * (c.field_h_mm - c.field_tol_mm));
    }
    *lo = l; *hi = h;
}

__global__ void k_gl_select(GlCfg c, const int* __restrict__ parent, const unsigned int* __restrict__ area, const unsigned int* __restrict__ bx0,
                            const unsigned int* __restrict__ bx1, const unsigned int* __restrict__ by0, const unsigned int* __restrict__ by1,
                            GlCand* __restrict__ cand, int* __restrict__ ncand) {
    const int f = blockIdx.y, HW = c.H * c.W;
    const size_t o = (size_t)f * HW;
    double lo, hi;
    gl_area_bounds(c, &lo, &hi);
    const double d2 = c.dpmm * c.dpmm;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        if (parent[o + i] != i) continue;
        const int x0 = bx0[o + i], x1 = bx1[o + i], y0 = by0[o + i], y1 = by1[o + i];
        // segmentation.clear_border(buffer_size = border - 1): any pixel in the outer `border` rows / columns
        if (x0 < c.border || y0 < c.border || x1 >= c.W - c.border || y1 >= c.H - c.border) continue;
        const double a = (double)area[o + i], bb = (double)(x1 - x0 + 1) * (double)(y1 - y0 + 1);
        // necessary: area <= area_filled <= bbox area
        if (!(lo < bb / d2) || !(a / d2 < hi)) continue;
        const int slot = atomicAdd(&ncand[f], 1);
        if (slot < GL_MAXCAND) { GlCand q; q.root = i; q.x0 = x0; q.y0 = y0; q.x1 = x1; q.y1 = y1; q.area = (int)area[o + i]; cand[(size_t)f * GL_MAXCAND + slot] = q; }
    }
}

// ------------------------------------------------------------------------------------------------ per-candidate analysis
// tile bytes: bit 0 = region mask, bit 1 = outside (reached by the flood), bit 2 = border pixel of the perimeter image
__device__ inline void gl_flood_outside(unsigned char* tile, int th, int tw) {
    const int tid = threadIdx.x;
    for (int i = tid; i < th * tw; i += GL_THREADS) {
        const int y = i / tw, x = i - y * tw;
        if ((y == 0 || x == 0 || y == th - 1 || x == tw - 1) && !(tile[i] & 1)) tile[i] |= 2;
    }
    __syncthreads();
    while (true) {
        int changed = 0;
        for (int y = tid; y < th; y += GL_THREADS) {
            unsigned char* r = tile + (size_t)y * tw;
            for (int x = 1; x < tw; x++) if (r[x] == 0 && (r[x - 1] & 2)) { r[x] = 2; changed = 1; }
            for (int x = tw - 2; x >= 0; x--) if (r[x] == 0 && (r[x + 1] & 2)) { r[x] = 2; changed = 1; }
        }
        __syncthreads();
        for (int x = tid; x < tw; x += GL_THREADS) {
            for (int y = 1; y < th; y++) if (tile[(size_t)y * tw + x] == 0 && (tile[(size_t)(y - 1) * tw + x] & 2)) { tile[(size_t)y * tw + x] = 2; changed = 1; }
            for (int y = th - 2; y >= 0; y--) if (tile[(size_t)y * tw + x] == 0 && (tile[(size_t)(y + 1) * tw + x] & 2)) { tile[(size_t)y * tw + x] = 2; changed = 1; }
        }
        if (!__syncthreads_or(changed)) break;
    }
}

__device__ inline double gl_block_sum(double v, double* red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    double t = 0;
    for (int k = 0; k < GL_THREADS / 32; k++) t += red[k];
    __syncthreads();
    return t;
}

// one candidate region: mask tile -> filled area, perimeter, conditions, moments -> accepted-region record (block-wide, uniform flow)
__device__ void gl_analyze_one(const GlCfg& c, int k, int f, const uint16_t* __restrict__ img, const int* __restrict__ par, const GlFrame& F,
                               const GlCand q, unsigned char* tile, double* red, int* s_hist50, epid_region* __restrict__ acc,
                               int* __restrict__ nacc, int acc_cap, int* __restrict__ overflow) {
    const int tid = threadIdx.x;
    const double PI = 3.141592653589793, d2 = c.dpmm * c.dpmm;
    const int bh = q.y1 - q.y0 + 1, bw = q.x1 - q.x0 + 1, th = bh + 2, tw = bw + 2;
    __syncthreads();
    for (int i = tid; i < th * tw; i += GL_THREADS) {
        const int ty = i / tw, tx = i - ty * tw;
        unsigned char m = 0;
        if (ty >= 1 && ty <= bh && tx >= 1 && tx <= bw) {
            int r = par[(q.y0 + ty - 1) * c.W + (q.x0 + tx - 1)];
            if (r >= 0) { const int p = par[r]; if (p != r) r = p; }
            m = r == q.root ? 1 : 0;
        }
        tile[i] = m;
    }
    __syncthreads();
    gl_flood_outside(tile, th, tw);
    double filled = 0;
    for (int i = tid; i < th * tw; i += GL_THREADS) filled += (tile[i] & 2) ? 0.0 : 1.0;
    filled = gl_block_sum(filled, red);
    const double bbox_area = (double)bh * (double)bw, fa = filled / d2;
    bool ok = true;
    if (c.conditions & C_SIZE_BB) ok = ok && (fmax(PI * ((c.radius_mm - c.tol_mm) * (c.radius_mm - c.tol_mm)), 2.0) < fa && fa < PI * ((c.radius_mm + c.tol_mm) * (c.radius_mm + c.tol_mm)));
    if (c.conditions & C_MODEST) ok = ok && (fmax(PI * (((c.bb_size_mm - 2) / 2) * ((c.bb_size_mm - 2) / 2)), 2.0) < fa && fa < PI * (((c.bb_size_mm + 2) / 2) * ((c.bb_size_mm + 2) / 2)));
    if (c.conditions & C_SQ_SIZE) { const double rs = fmax(c.rad_size_mm, 5.0); ok = ok && ((rs - 5) * (rs - 5) < fa && fa < (rs + 5) * (rs + 5)); }
    if (c.conditions & C_AREA_SQ) ok = ok && ((c.field_w_mm - c.field_tol_mm) * (c.field_h_mm - c.field_tol_mm) < fa && fa < (c.field_w_mm + c.field_tol_mm) * (c.field_h_mm + c.field_tol_mm));
    const double ratio = filled / bbox_area;
    if (c.conditions & C_ROUND) ok = ok && (PI / 4 * 1.2 > ratio && ratio > PI / 4 * 0.8);
    if (c.conditions & C_SQUARE) ok = ok && (ratio > 0.8);
    if (c.conditions & C_SYM) { const double y = (double)bh, x = (double)bw; ok = ok && !(x > fmax(y * 1.05, y + 3) || x < fmin(y * 0.95, y - 3)); }
    if (!ok) return;      // uniform: every quantity above is block-wide
    // skimage.measure.perimeter(region.image, neighborhood=4)
    if (tid < 50) s_hist50[tid] = 0;
    __syncthreads();
    for (int i = tid; i < th * tw; i += GL_THREADS) {
        if (!(tile[i] & 1)) continue;
        const bool er = (tile[i - 1] & 1) && (tile[i + 1] & 1) && (tile[i - tw] & 1) && (tile[i + tw] & 1);      // the margin guarantees neighbours
        if (!er) tile[i] |= 4;
    }
    __syncthreads();
    for (int i = tid; i < th * tw; i += GL_THREADS) {
        const int ty = i / tw, tx = i - ty * tw;
        int v = 0;
        for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) {
                const int yy = ty + dy, xx = tx + dx;
                if (yy < 0 || yy >= th || xx < 0 || xx >= tw) continue;
                if (tile[yy * tw + xx] & 4) v += (dy == 0 && dx == 0) ? 1 : ((dy == 0 || dx == 0) ? 2 : 10);
            }
        if (v > 0 && v < 50) atomicAdd(&s_hist50[v], 1);
    }
    __syncthreads();
    double perim = 0.0;
    {
        const double w1 = 1.0, w2 = sqrt(2.0), w3 = (1 + sqrt(2.0)) / 2;
        for (int b = 0; b < 50; b++) {
            double wk = 0.0;
            if (b == 5 || b == 7 || b == 15 || b == 17 || b == 25 || b == 27) wk = w1;
            else if (b == 21 || b == 33) wk = w2;
            else if (b == 13 || b == 23) wk = w3;
            perim += (double)s_hist50[b] * wk;
        }
    }
    __syncthreads();
    const double per_mm = perim / c.dpmm;
    if (c.conditions & C_CIRC) ok = ok && (2 * PI * (c.radius_mm + c.tol_mm) > per_mm && per_mm > 2 * PI * (c.radius_mm - c.tol_mm));
    if (c.conditions & C_SQ_PERIM) {
        const double up = 1.20 * 2 * (c.field_w_mm + c.field_tol_mm) + 2 * (c.field_h_mm + c.field_tol_mm);
        const double lw = 2 * (c.field_w_mm - c.field_tol_mm) + 2 * (c.field_h_mm - c.field_tol_mm);
        ok = ok && (up > per_mm && per_mm > lw);
    }
    if (!ok) return;
    // accepted: centroid, weighted centroid (weights = the sample values), equivalent diameter
    double sw = 0, swr = 0, swc = 0, sr = 0, sc = 0;
    const unsigned int D = F.mx - F.mn;
    for (int i = tid; i < bh * bw; i += GL_THREADS) {
        const int r = i / bw, cidx = i - r * bw;
        if (!(tile[(r + 1) * tw + (cidx + 1)] & 1)) continue;
        const double wv = gl_sample(c.mode, c.kind, c.invert, img[(q.y0 + r) * c.W + (q.x0 + cidx)], F.mn, D);
        sw += wv; swr += (double)r * wv; swc += (double)cidx * wv;
        sr += (double)r; sc += (double)cidx;
    }
    sw = gl_block_sum(sw, red); swr = gl_block_sum(swr, red); swc = gl_block_sum(swc, red);
    sr = gl_block_sum(sr, red); sc = gl_block_sum(sc, red);
    if (tid == 0) {
        const int slot = atomicAdd(&nacc[f], 1);
        if (slot < acc_cap) {
            epid_region R;
            R.threshold_index = k;
            R.label_root = q.root;
            R.area = (double)q.area;
            R.area_filled = filled;
            R.perimeter = perim;
            R.bbox[0] = q.y0; R.bbox[1] = q.x0; R.bbox[2] = q.y1 + 1; R.bbox[3] = q.x1 + 1;
            R.centroid_y = sr / (double)q.area + (double)q.y0;
            R.centroid_x = sc / (double)q.area + (double)q.x0;
            R.wcentroid_y = swr / sw + (double)q.y0;
            R.wcentroid_x = swc / sw + (double)q.x0;
            R.equivalent_diameter = sqrt(4 * (double)q.area / PI);
            acc[(size_t)f * acc_cap + slot] = R;
        } else atomicOr(&overflow[f], 2);
    }
}

__global__ void __launch_bounds__(GL_THREADS)
k_gl_analyze(GlCfg c, int role, const uint16_t* __restrict__ frames, const GlFrame* __restrict__ gf, int k, const int* __restrict__ parent,
             const GlCand* __restrict__ cand, const int* __restrict__ ncand, unsigned char* __restrict__ big_tiles, epid_region* __restrict__ acc,
             int* __restrict__ nacc, int acc_cap, int* __restrict__ overflow) {
    extern __shared__ __align__(16) unsigned char sm_tile[];
    __shared__ double red[GL_THREADS / 32];
    __shared__ int s_hist50[50];
    const int f = blockIdx.y, HW = c.H * c.W;
    const int nc = min(ncand[f], GL_MAXCAND);
    if (ncand[f] > GL_MAXCAND && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&overflow[f], 1);
    const GlFrame& F = gf[f];
    const uint16_t* img = frames + (size_t)f * HW;
    const int* par = parent + (size_t)f * HW;
    auto tile_bytes = [](const GlCand& q) { return (size_t)(q.y1 - q.y0 + 3) * (size_t)(q.x1 - q.x0 + 3); };
    // role 0 (small shared tile): the candidates whose tile fits GL_SMALL_TILE, round-robin over the CTAs of the frame;
    // role 1 (large shared tile): the candidates between the two capacities, round-robin; CTA 0 then takes, one after the other, the
    // candidates beyond the large tile (tile in HBM scratch)
    for (int ci = blockIdx.x; ci < nc; ci += gridDim.x) {
        const GlCand q = cand[(size_t)f * GL_MAXCAND + ci];
        const size_t tb = tile_bytes(q);
        if (role == 0 ? tb > (size_t)GL_SMALL_TILE : (tb <= (size_t)GL_SMALL_TILE || tb > (size_t)GL_TILE_BYTES)) continue;
        gl_analyze_one(c, k, f, img, par, F, q, sm_tile, red, s_hist50, acc, nacc, acc_cap, overflow);
    }
    if (role == 1 && blockIdx.x == 0) {
        unsigned char* big = big_tiles + (size_t)f * (size_t)(c.H + 2) * (c.W + 2);
        for (int ci = 0; ci < nc; ci++) {
            const GlCand q = cand[(size_t)f * GL_MAXCAND + ci];
            if (tile_bytes(q) <= (size_t)GL_TILE_BYTES) continue;
            gl_analyze_one(c, k, f, img, par, F, q, big, red, s_hist50, acc, nacc, acc_cap, overflow);
        }
    }
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_global_locate(epid_ctx* ctx, const epid_batch* frames, const epid_locate_params* p, epid_region* regions,
                                      int32_t region_cap, int32_t* counts, int32_t* flags) {
    EPID_REQUIRE(ctx && frames && p && regions && counts && flags && region_cap > 0, EPID_ERR_INVALID, "NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device"); return EPID_ERR_NO_DEVICE; }
    EPID_REQUIRE(frames->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "the global locators need uint16 frames");
    EPID_REQUIRE(p->mode == 0 || p->mode == 1, EPID_ERR_INVALID, "mode 0 (disk) or 1 (field)");
    EPID_REQUIRE(!(p->conditions & C_SOLID), EPID_ERR_UNSUPPORTED, "is_solid is not available in the whole-frame finder");
    EPID_REQUIRE(p->dpmm > 0, EPID_ERR_INVALID, "dpmm must be positive");
    EPID_CUDA(cudaSetDevice(ctx->device));
    if (frames->n > GL_CHUNK) {
        // 24 B of labelling scratch per pixel and frame: large batches run in chunks of GL_CHUNK frames
        for (int c0 = 0; c0 < frames->n; c0 += GL_CHUNK) {
            epid_batch sub = *frames;
            sub.owns = false;
            sub.n = std::min(GL_CHUNK, frames->n - c0);
            sub.dptr = (char*)frames->dptr + (size_t)c0 * frames->h * frames->w * sizeof(uint16_t);
            const int rc = epid_global_locate(ctx, &sub, p, regions + (size_t)c0 * region_cap, region_cap, counts + c0, flags + c0);
            if (rc != EPID_OK) return rc;
        }
        return EPID_OK;
    }
    const int n = frames->n, H = frames->h, W = frames->w, HW = H * W;
    EPID_REQUIRE((size_t)H * W < (1u << 30), EPID_ERR_UNSUPPORTED, "frame too large");
    GlCfg c;
    c.mode = p->mode; c.kind = p->sample_kind; c.invert = p->invert; c.conn8 = p->mode == 1 ? 1 : 0;
    c.border = p->mode == 1 ? 4 : 1;      // clear_border(buffer_size=3) removes the outer 4 rows / columns; buffer_size=0 the outer 1
    c.conditions = p->conditions; c.H = H; c.W = W; c.dpmm = p->dpmm;
    c.radius_mm = p->radius_mm; c.tol_mm = p->tolerance_mm; c.field_w_mm = p->field_width_mm; c.field_h_mm = p->field_height_mm;
    c.field_tol_mm = p->field_tolerance_mm; c.bb_size_mm = p->bb_size_mm; c.rad_size_mm = p->rad_size_mm;
    auto rup = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t b_gf = rup(sizeof(GlFrame) * n), b_par = rup(sizeof(int) * (size_t)n * HW), b_prop = rup(sizeof(unsigned int) * (size_t)n * HW);
    const size_t b_cand = rup(sizeof(GlCand) * (size_t)n * GL_MAXCAND), b_cnt = rup(sizeof(int) * n);
    const size_t b_big = rup((size_t)n * (H + 2) * (W + 2)), b_acc = rup(sizeof(epid_region) * (size_t)n * region_cap);
    int rc = ensure_scratch(ctx, b_gf + b_par + 5 * b_prop + b_cand + 3 * b_cnt + b_big + b_acc + 1024);
    if (rc != EPID_OK) return rc;
    char* q = (char*)ctx->scratch;
    GlFrame* d_gf = (GlFrame*)q; q += b_gf;
    int* d_par = (int*)q; q += b_par;
    unsigned int* d_area = (unsigned int*)q; q += b_prop;
    unsigned int* d_x0 = (unsigned int*)q; q += b_prop;
    unsigned int* d_x1 = (unsigned int*)q; q += b_prop;
    unsigned int* d_y0 = (unsigned int*)q; q += b_prop;
    unsigned int* d_y1 = (unsigned int*)q; q += b_prop;
    GlCand* d_cand = (GlCand*)q; q += b_cand;
    int* d_ncand = (int*)q; q += b_cnt;
    int* d_nacc = (int*)q; q += b_cnt;
    int* d_over = (int*)q; q += b_cnt;
    unsigned char* d_big = (unsigned char*)q; q += b_big;
    epid_region* d_acc = (epid_region*)q;
    const uint16_t* fr = (const uint16_t*)frames->dptr;
    EPID_SMEM_OPT_IN(ctx, k_gl_analyze, GL_TILE_BYTES);
    EPID_CUDA(cudaMemsetAsync(d_nacc, 0, sizeof(int) * n, ctx->stream));
    EPID_CUDA(cudaMemsetAsync(d_over, 0, sizeof(int) * n, ctx->stream));
    k_gl_minmax_init<<<(n + 127) / 128, 128, 0, ctx->stream>>>(d_gf, n);
    k_gl_minmax<<<dim3(64, n), 256, 0, ctx->stream>>>(fr, (size_t)HW, d_gf);
    k_gl_plan<<<(n + 63) / 64, 64, 0, ctx->stream>>>(d_gf, n, c.mode, c.kind, c.invert);
    ctx->launches += 3;
    const int nthr_max = c.mode == 0 ? 50 : 46;
    const dim3 g(ctx->sm_count * 2, n);
    for (int k = 0; k < nthr_max; k++) {
        k_gl_init<<<g, 256, 0, ctx->stream>>>(fr, HW, d_gf, k, d_par, d_ncand);
        k_ccl_union<<<g, 256, 0, ctx->stream>>>(H, W, c.conn8, d_par);
        k_gl_flatten<<<g, 256, 0, ctx->stream>>>(HW, W, H, d_par, d_area, d_x0, d_x1, d_y0, d_y1);
        k_gl_props<<<g, 256, 0, ctx->stream>>>(HW, W, d_par, d_area, d_x0, d_x1, d_y0, d_y1);
        k_gl_select<<<g, 256, 0, ctx->stream>>>(c, d_par, d_area, d_x0, d_x1, d_y0, d_y1, d_cand, d_ncand);
        k_gl_analyze<<<dim3(128, n), GL_THREADS, GL_SMALL_TILE, ctx->stream>>>(c, 0, fr, d_gf, k, d_par, d_cand, d_ncand, d_big, d_acc, d_nacc,
                                                                            region_cap, d_over);
        k_gl_analyze<<<dim3(8, n), GL_THREADS, GL_TILE_BYTES, ctx->stream>>>(c, 1, fr, d_gf, k, d_par, d_cand, d_ncand, d_big, d_acc, d_nacc,
                                                                          region_cap, d_over);
        ctx->launches += 7;  // init, union, flatten, props, select, analyze x 2
        if (getenv("EPID_DEBUG_LOCATE")) {      // diagnostics: per threshold the plan, candidates and accepted regions of frame 0
            GlFrame hf;
            int hc = 0, ha = 0;
            cudaMemcpyAsync(&hf, d_gf, sizeof(hf), cudaMemcpyDeviceToHost, ctx->stream);
            cudaMemcpyAsync(&hc, d_ncand, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
            cudaMemcpyAsync(&ha, d_nacc, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
            cudaError_t e = cudaStreamSynchronize(ctx->stream);
            std::vector<int> hp((size_t)HW);
            cudaMemcpy(hp.data(), d_par, sizeof(int) * (size_t)HW, cudaMemcpyDeviceToHost);
            long fg = 0, roots = 0;
            for (int i = 0; i < HW; i++) { fg += hp[i] >= 0; roots += hp[i] == i; }
            fprintf(stderr, "[locate] k %d (%s) mn %u mx %u nthr %d dir %d T %u cutoff %g fg %ld roots %ld ncand %d nacc %d\n", k, cudaGetErrorString(e), hf.mn,
                    hf.mx, hf.nthr, k < GL_MAXTHR ? hf.dir[k] : 0, k < GL_MAXTHR ? hf.T[k] : 0u, k < GL_MAXTHR ? hf.cutoff[k] : 0.0, fg, roots, hc, ha);
        }
    }
    EPID_CUDA(cudaGetLastError());
    std::vector<int> h_n(n), h_o(n);
    EPID_CUDA(cudaMemcpyAsync(h_n.data(), d_nacc, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(h_o.data(), d_over, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(regions, d_acc, sizeof(epid_region) * (size_t)n * region_cap, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int f = 0; f < n; f++) {
        counts[f] = std::min(h_n[f], region_cap);
        flags[f] = h_o[f];
        // the reference's order: threshold, then label (raster position of the region's first pixel)
        epid_region* r = regions + (size_t)f * region_cap;
        std::sort(r, r + counts[f], [](const epid_region& a, const epid_region& b) {
            return a.threshold_index != b.threshold_index ? a.threshold_index < b.threshold_index : a.label_root < b.label_root;
        });
    }
    return EPID_OK;
}
