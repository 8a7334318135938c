// CT phantom localization (pylinac.ct, ct.py:381-433 Slice.phantom_roi with ct.py:3315-3348 get_regions: fill_holes=True,
// threshold="otsu"), for every listed slice of a device-resident int16 / uint16 series, on both branches of get_regions:
//   ndarray branch (clip_in_localization=True):  Otsu of every pixel of the smoothed edges of np.clip(HU, -1000, 1000)
//   Slice branch (clip_in_localization=False):   Otsu of the pixels of skimage.draw.disk(image centre, radius) of the smoothed edges
//                                                of the unclipped HU, times 0.8 (radius = 110 mm in pixels)
// and epid_ct_regions, the region table of get_regions(slice) with its defaults (Slice branch, no hole filling, borders cleared) for
// one slice, which CatPhanBase.find_phantom_roll (ct.py:2522-2563) reads.
//
// Per slice, each stage equal bit for bit to the numpy / scipy / skimage call it restates:
//   k_ct_scharr   HU = raw * slope + intercept (float64, two roundings), skimage.filters.scharr of HU (its maximum: the edge check)
//                 and, on the ndarray branch, of np.clip(HU, -1000, 1000), each ndimage.convolve pass in NI_Correlate's footprint
//                 order, mode 'reflect'
//   correlate1d   skimage.filters.gaussian(sigma=1) = ndimage.gaussian_filter(mode='nearest', truncate=4): filters.cu's passes
//   k_ct_otsu     threshold_otsu: np.histogram's 256 linspace bins and float bin assignment, then the between-class variance argmax
//   k_ct_*        bw = edges > thres; clear_border (8-connected objects reaching the outer buffer_size + 1 rows / columns);
//                 binary_fill_holes (background 4-connected to the outside stays); measure.label (8-connected); per region the
//                 area and exact row / column sums
//   k_ct_select   the region with the smallest |area - catphan_size| (first label on ties) and the 1.3x size check
//   k_ct_region_* per region of the unfilled mask (epid_ct_regions): bbox, exact first and second moments, and filled_area, the
//                 binary_fill_holes of the region's own bbox crop
// Labels are union-find roots within each slice (ccl.cuh): the smallest index of a component, which is skimage's raster label order.
// After the global fill every region's filled_area equals its area (no background is enclosed), so area stands for both.
#include <cfloat>
#include <cstring>

#include "ccl.cuh"
#include "common.cuh"
#include "filters.cuh"
#include "roi.cuh"

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

// E: the edges the Gaussian smooths, the Scharr of the clipped HU (CLIP: the ndarray branch) or of the HU itself (the Slice branch)
template <typename T, bool CLIP>
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
                if (CLIP) c[j * 3 + i] = fmin(fmax(h, -1000.0), 1000.0);
            }
        e = scharr3(v);
        E[((size_t)s * H + y) * W + x] = CLIP ? scharr3(c) : e;
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

// The pixels k_ct_otsu reads on the Slice branch: skimage.draw.disk(centre, R, shape) -- roi.cuh's disk_box clipped to the slice,
// rows r0 .. r0 + bh - 1 and columns c0 .. c0 + bw - 1, and the member test of the float offsets from the clipped box's corner,
// ((i - sr) / R)**2 + ((j - sc) / R)**2 < 1 with (sr, sc) = centre - corner.  The centre (H / 2 - 0.5, W / 2 - 0.5) is a
// half-integer or an integer, so i - sr is the pixel's exact offset from the centre wherever the corner lies: clipping drops the
// pixels outside the slice and changes no member test of the others.
struct OtsuDisk {
    int r0, c0, bh, bw;
    double sr, sc, R;
};

// pixel k of what threshold_otsu reads: the whole slice (p = k), or (DISK) box pixel k in raster order, false if not a member
template <bool DISK>
__device__ __forceinline__ bool otsu_pixel(const OtsuDisk& d, int W, int k, int& p) {
    if (!DISK) { p = k; return true; }
    const int i = k / d.bw, j = k - i * d.bw;
    p = (d.r0 + i) * W + d.c0 + j;
    const double a = ((double)i - d.sr) / d.R, b = ((double)j - d.sc) / d.R;
    return a * a + b * b < 1.0;
}

// threshold_otsu of each slice's S (one CTA per slice): of every pixel, or (DISK) of the disk's pixels times 0.8.  Only membership
// matters: min, max and the histogram are order-free, and np.all(x == x[0]) is min == max (no edge plane holds a NaN).
template <bool DISK>
__global__ void __launch_bounds__(CT_SEL_THREADS)
k_ct_otsu(const double* __restrict__ S, int HW, int W, OtsuDisk disk, double* __restrict__ thres) {
    __shared__ double rmn[32], rmx[32];
    __shared__ double edge[CT_BINS + 1];
    __shared__ unsigned int hist[CT_BINS];
    __shared__ double cum_hi[CT_BINS];
    __shared__ long long w2[CT_BINS];
    const double* f = S + (size_t)blockIdx.x * HW;
    const int n = DISK ? disk.bh * disk.bw : HW;
    const double scale = DISK ? 0.8 : 1.0;
    double mn = INFINITY, mx = -INFINITY;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        int i;
        if (!otsu_pixel<DISK>(disk, W, k, i)) continue;
        const double v = f[i]; mn = fmin(mn, v); mx = fmax(mx, v);
    }
    mn = warp_min(mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { rmn[threadIdx.x >> 5] = mn; rmx[threadIdx.x >> 5] = mx; }
    for (int i = threadIdx.x; i < CT_BINS; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    mn = rmn[0]; mx = rmx[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) { mn = fmin(mn, rmn[k]); mx = fmax(mx, rmx[k]); }
    if (mn == mx) {                       // np.all(image == first_pixel): the threshold is that value
        if (threadIdx.x == 0) thres[blockIdx.x] = DISK ? mn * scale : mn;
        return;
    }
    // np.linspace(mn, mx, 257): i * step + start, the last edge exactly mx
    const double step = (mx - mn) / (double)CT_BINS;
    for (int i = threadIdx.x; i <= CT_BINS; i += blockDim.x) edge[i] = i == CT_BINS ? mx : (double)i * step + mn;
    __syncthreads();
    const double denom = mx - mn;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        int i;
        if (!otsu_pixel<DISK>(disk, W, k, i)) continue;
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
    const double t = (edge[arg] + edge[arg + 1]) / 2.0;
    thres[blockIdx.x] = DISK ? t * scale : t;
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


// ---------------------------------------------------------------------------------- the region table of get_regions(slice)
// One slice, P its labelled mask (roots).  Per root: the bbox by atomic min / max, then the second moments about the bbox corner.

__global__ void k_ct_region_bbox(int W, int HW, const int* __restrict__ P, int* __restrict__ box) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW || P[p] < 0) return;
    const int r = P[p], y = p / W, x = p - y * W;
    atomicMin(&box[r], y);
    atomicMin(&box[HW + r], x);
    atomicMax(&box[2 * HW + r], y + 1);
    atomicMax(&box[3 * HW + r], x + 1);
}

__global__ void k_ct_region_moments(int W, int HW, const int* __restrict__ P, const int* __restrict__ box,
                                    unsigned long long* __restrict__ mom) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW || P[p] < 0) return;
    const int r = P[p], y = p / W, x = p - y * W;
    const unsigned long long dy = (unsigned long long)(y - box[r]), dx = (unsigned long long)(x - box[HW + r]);
    if (dy) atomicAdd(&mom[r], dy * dy);
    if (dx) atomicAdd(&mom[HW + r], dx * dx);
    if (dy && dx) atomicAdd(&mom[2 * HW + r], dy * dx);
}

// The rows in label order (one CTA): the roots in raster order, compacted a block of pixels at a time; the first `cap` are written,
// `count` gets them all.  filled_area is left to k_ct_region_fill.
__global__ void __launch_bounds__(CT_SEL_THREADS)
k_ct_region_rows(int HW, const int* __restrict__ P, const unsigned int* __restrict__ area, const unsigned long long* __restrict__ rsum,
                 const unsigned long long* __restrict__ csum, const int* __restrict__ box, const unsigned long long* __restrict__ mom,
                 int cap, epid_ct_region* __restrict__ rows, int* __restrict__ count) {
    __shared__ int wsum[32];
    __shared__ int s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    for (int p0 = 0; p0 < HW; p0 += blockDim.x) {
        const int p = p0 + threadIdx.x;
        const bool root = p < HW && P[p] == p;
        const unsigned bal = __ballot_sync(0xffffffffu, root);
        if (lane == 0) wsum[warp] = __popc(bal);
        __syncthreads();
        int k = s_base + __popc(bal & ((1u << lane) - 1u));
        for (int w = 0; w < warp; w++) k += wsum[w];
        if (root && k < cap) {
            epid_ct_region& o = rows[k];
            o.label = k + 1;
            o.first = p;
            o.area = (int32_t)area[p];
            o.filled_area = 0;
            for (int j = 0; j < 4; j++) o.bbox[j] = box[j * HW + p];
            o.sum_r = rsum[p];
            o.sum_c = csum[p];
            o.m_rr = mom[p];
            o.m_cc = mom[HW + p];
            o.m_rc = mom[2 * HW + p];
        }
        __syncthreads();
        if (threadIdx.x == 0)
            for (int w = 0; w < nwarps; w++) s_base += wsum[w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = s_base;
}

// filled_area of row blockIdx.x: skimage's binary_fill_holes of the region's own bbox crop (4-connected background; other regions'
// pixels are background).  The crop's background is a bitmask C (bit b of word xw of row y: column 32 xw + b), and F its part
// 4-connected to the crop's border: seeded with C's border pixels and dilated in place -- across words by the neighbouring words,
// within a word by shifts until it stops changing -- until no word changes.  F only grows and stays inside the true flood, so reading
// a neighbour word mid-update is harmless, and a sweep in which no thread changed a word is the fixed point.
// filled_area = crop pixels - |F|.  ws: C then F, at word offset off[row].
__global__ void __launch_bounds__(CT_THREADS)
k_ct_region_fill(int W, const int* __restrict__ P, epid_ct_region* __restrict__ rows, const long long* __restrict__ off,
                 unsigned int* __restrict__ ws) {
    __shared__ unsigned long long red[32];
    epid_ct_region& r = rows[blockIdx.x];
    const int r0 = r.bbox[0], c0 = r.bbox[1], h = r.bbox[2] - r0, w = r.bbox[3] - c0, root = r.first;
    const int wr = (w + 31) >> 5, nw = h * wr;
    unsigned int* C = ws + off[blockIdx.x];
    unsigned int* F = C + nw;
    for (int q = threadIdx.x; q < nw; q += blockDim.x) {
        const int y = q / wr, xw = q - y * wr;
        const int* row = P + (size_t)(r0 + y) * W + c0;
        unsigned int c = 0;
        for (int b = 0; b < 32; b++) {
            const int x = xw * 32 + b;
            if (x < w && row[x] != root) c |= 1u << b;
        }
        unsigned int border = (y == 0 || y == h - 1) ? ~0u : 0u;
        if (xw == 0) border |= 1u;
        if (xw == wr - 1) border |= 1u << ((w - 1) & 31);
        C[q] = c;
        F[q] = c & border;
    }
    __syncthreads();
    while (true) {
        int changed = 0;
        for (int q = threadIdx.x; q < nw; q += blockDim.x) {
            const unsigned int c = C[q];
            if (!c) continue;
            const int y = q / wr, xw = q - y * wr;
            const unsigned int f = F[q];
            unsigned int x = f | (f << 1) | (f >> 1);
            if (y > 0) x |= F[q - wr];
            if (y < h - 1) x |= F[q + wr];
            if (xw > 0) x |= F[q - 1] >> 31;
            if (xw < wr - 1) x |= F[q + 1] << 31;
            x &= c;
            for (;;) {
                const unsigned int g = c & (x | (x << 1) | (x >> 1));
                if (g == x) break;
                x = g;
            }
            if (x != f) { F[q] = x; changed = 1; }
        }
        if (!__syncthreads_or(changed)) break;
    }
    unsigned long long flooded = 0;
    for (int q = threadIdx.x; q < nw; q += blockDim.x) flooded += __popc(F[q]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) flooded += __shfl_xor_sync(0xffffffffu, flooded, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = flooded;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); k++) t += red[k];
        r.filled_area = (int32_t)((long long)h * w - (long long)t);
    }
}

inline unsigned blocks(int N) { return (unsigned)((N + CT_THREADS - 1) / CT_THREADS); }

// The device planes of one chunk of m slices (every plane m * H * W)
struct CtPlanes {
    SliceIn* in;
    unsigned long long* emax;
    double* thr;
    double *E, *T, *S;
    int *P, *Q, *flag;
    uint8_t* F;
};

// The stage sequence both entries share, for the m slices staged in c.in: the Scharr edges and edge maxima, the Gaussian, Otsu over
// every pixel (disk NULL) or over the disk (the Slice branch), bw = smoothed > threshold, clear_border, binary_fill_holes (fill) and
// 8-connected labelling, leaving slice-local roots in c.P.  Returns the first error; a CUDA error is left in e.
int ct_label_chunk(epid_ctx* ctx, int dtype, const CtPlanes& c, int m, int H, int W, bool clear_borders, const OtsuDisk* disk,
                   bool fill, const double* gauss_w, int gauss_r, cudaError_t& e) {
    const long long HW = (long long)H * W;
    const int N = (int)(HW * m);
    const dim3 g_scharr((W + CT_THREADS - 1) / CT_THREADS, H, m);
    const dim3 g_union(blocks((int)HW), m);      // one thread per pixel, slices in grid.y
    // clear_border's band: buffer_size = min(int(max(H, W) / 100), 3) rows / columns plus one
    const int ext = std::min((int)((double)std::max(H, W) / 100.0), 3) + 1;
    e = cudaMemsetAsync(c.emax, 0, 8 * m, ctx->stream);
    if (e != cudaSuccess) return EPID_OK;
    if (dtype == EPID_I16) {
        if (disk) k_ct_scharr<int16_t, false><<<g_scharr, CT_THREADS, 0, ctx->stream>>>(c.in, H, W, c.E, c.emax);
        else k_ct_scharr<int16_t, true><<<g_scharr, CT_THREADS, 0, ctx->stream>>>(c.in, H, W, c.E, c.emax);
    } else {
        if (disk) k_ct_scharr<uint16_t, false><<<g_scharr, CT_THREADS, 0, ctx->stream>>>(c.in, H, W, c.E, c.emax);
        else k_ct_scharr<uint16_t, true><<<g_scharr, CT_THREADS, 0, ctx->stream>>>(c.in, H, W, c.E, c.emax);
    }
    int rc = correlate1d_f64(ctx, c.E, c.T, m, H, W, 0, gauss_w, gauss_r, 1);
    if (rc == EPID_OK) rc = correlate1d_f64(ctx, c.T, c.S, m, H, W, 1, gauss_w, gauss_r, 1);
    if (rc != EPID_OK) return rc;
    if (disk) k_ct_otsu<true><<<m, CT_SEL_THREADS, 0, ctx->stream>>>(c.S, (int)HW, W, *disk, c.thr);
    else k_ct_otsu<false><<<m, CT_SEL_THREADS, 0, ctx->stream>>>(c.S, (int)HW, W, OtsuDisk{}, c.thr);
    k_ct_binarize<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(c.S, c.thr, (int)HW, N, c.P);
    ctx->launches += 3;
    if (clear_borders) {
        k_ccl_union<<<g_union, CT_THREADS, 0, ctx->stream>>>(H, W, 1, c.P);
        k_ct_flatten<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, c.P);
        e = cudaMemsetAsync(c.flag, 0, 4 * N, ctx->stream);
        if (e != cudaSuccess) return EPID_OK;
        k_ct_mark_border<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(H, W, N, ext, c.P, c.flag);
        k_ct_clear_flagged<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, c.P, c.flag);
        ctx->launches += 4;
    }
    if (fill) {
        k_ct_background<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, c.P, c.Q);
        k_ccl_union<<<g_union, CT_THREADS, 0, ctx->stream>>>(H, W, 0, c.Q);
        k_ct_flatten<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, c.Q);
        e = cudaMemsetAsync(c.flag, 0, 4 * N, ctx->stream);
        if (e != cudaSuccess) return EPID_OK;
        k_ct_mark_border<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(H, W, N, 1, c.Q, c.flag);
        k_ct_fill<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, c.P, c.Q, c.flag, c.F);
        ctx->launches += 5;
    }
    k_ccl_union<<<g_union, CT_THREADS, 0, ctx->stream>>>(H, W, 1, c.P);
    k_ct_flatten<<<blocks(N), CT_THREADS, 0, ctx->stream>>>((int)HW, N, c.P);
    ctx->launches += 2;
    e = cudaGetLastError();
    return EPID_OK;
}

// The common argument checks; on success the Otsu disk of the Slice branch (disk_r > 0) is in *disk and *use_disk is set
int ct_check(epid_ctx* ctx, const epid_batch* volume, const double* slope, const double* intercept, int32_t clip_in_localization,
             double disk_r, const double* gauss_w, int32_t gauss_r, OtsuDisk* disk, bool* use_disk) {
    EPID_REQUIRE(ctx && volume && slope && intercept && gauss_w, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(clip_in_localization || disk_r > 0, EPID_ERR_UNSUPPORTED,
                 "localization without clipping needs the Otsu disk of a Slice passed to get_regions (otsu_disk_radius > 0)");
    EPID_REQUIRE(!clip_in_localization || !(disk_r > 0), EPID_ERR_INVALID,
                 "an Otsu disk (otsu_disk_radius > 0: a Slice passed to get_regions) is not clipped; clip_in_localization must be 0");
    EPID_REQUIRE(volume->dtype == EPID_I16 || volume->dtype == EPID_U16, EPID_ERR_UNSUPPORTED,
                 "CT localization reads int16 or uint16 slices");
    EPID_REQUIRE(gauss_r >= 0, EPID_ERR_INVALID, "bad Gaussian radius");
    const int H = volume->h, W = volume->w;
    // the kernels put a slice's rows in grid.y
    EPID_REQUIRE(H >= 2 && W >= 2 && H <= CT_MAX_GRID && (long long)H * W <= CT_CHUNK_PIXELS, EPID_ERR_UNSUPPORTED,
                 "slices of %d x %d pixels are not supported (at least 2 x 2, at most %d rows and %lld pixels)", H, W, CT_MAX_GRID,
                 CT_CHUNK_PIXELS);
    *use_disk = disk_r > 0;
    if (*use_disk) {
        // a radius of at least 1 holds the pixels nearest the centre, so threshold_otsu never sees an empty disk
        EPID_REQUIRE(disk_r >= 1.0 && std::isfinite(disk_r), EPID_ERR_INVALID, "otsu_disk_radius %g is below 1 pixel", disk_r);
        const double cy = H / 2.0 - 0.5, cx = W / 2.0 - 0.5;
        const DiskBox b = disk_box(cy, cx, disk_r);
        const long long r0 = std::max(b.r0, 0ll), c0 = std::max(b.c0, 0ll);
        const long long r1 = std::min(b.r0 + b.bh - 1, (long long)H - 1), c1 = std::min(b.c0 + b.bw - 1, (long long)W - 1);
        *disk = OtsuDisk{(int)r0, (int)c0, (int)(r1 - r0 + 1), (int)(c1 - c0 + 1), cy - (double)r0, cx - (double)c0, disk_r};
    }
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_ct_localize(epid_ctx* ctx, const epid_batch* volume, const double* slope, const double* intercept,
                                    const int32_t* slices, int32_t nslices, double catphan_size, int32_t clear_borders,
                                    int32_t clip_in_localization, double otsu_disk_radius, const double* gauss_w, int32_t gauss_r,
                                    struct epid_ct_slice* results, double* scharr, double* smoothed, uint8_t* filled, int32_t* labels) {
    EPID_REQUIRE(slices && results, EPID_ERR_INVALID, "NULL argument");
    OtsuDisk disk{};
    bool use_disk = false;
    const int rc0 = ct_check(ctx, volume, slope, intercept, clip_in_localization, otsu_disk_radius, gauss_w, gauss_r, &disk, &use_disk);
    if (rc0 != EPID_OK) return rc0;
    EPID_REQUIRE(nslices >= 0, EPID_ERR_INVALID, "bad slice count");
    const int H = volume->h, W = volume->w;
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
    CtPlanes c;
    c.in = (SliceIn*)(d + o_in);
    c.emax = (unsigned long long*)(d + o_emax);
    c.thr = (double*)(d + o_thr);
    c.E = (double*)(d + o_E); c.T = (double*)(d + o_T); c.S = (double*)(d + o_S);
    c.P = (int*)(d + o_P); c.Q = (int*)(d + o_Q); c.flag = (int*)(d + o_A);
    c.F = (uint8_t*)(d + o_F);
    epid_ct_slice* d_rows = (epid_ct_slice*)(d + o_rows);
    unsigned int* A = (unsigned int*)(d + o_A);
    unsigned long long *R = (unsigned long long*)(d + o_R), *Cs = (unsigned long long*)(d + o_C);

    std::vector<SliceIn> hin(chunk);
    cudaError_t e = cudaSuccess;
    int rc = EPID_OK;
    for (int k0 = 0; k0 < nslices && rc == EPID_OK && e == cudaSuccess; k0 += chunk) {
        const int m = std::min(chunk, nslices - k0);
        const int N = (int)(HW * m);
        for (int j = 0; j < m; j++) {
            const int sl = slices[k0 + j];
            hin[j] = SliceIn{(const char*)volume->dptr + (size_t)sl * HW * esz, slope[sl], intercept[sl]};
        }
        // the inputs are staged from host memory that changes per chunk: copy synchronously with respect to the host
        e = cudaMemcpyAsync(c.in, hin.data(), sizeof(SliceIn) * m, cudaMemcpyHostToDevice, ctx->stream);
        if (e != cudaSuccess) break;
        rc = ct_label_chunk(ctx, volume->dtype, c, m, H, W, clear_borders, use_disk ? &disk : nullptr, true, gauss_w, gauss_r, e);
        if (rc != EPID_OK || e != cudaSuccess) break;
        e = cudaMemsetAsync(A, 0, 4 * N, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(R, 0, 8 * N, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(Cs, 0, 8 * N, ctx->stream);
        if (e != cudaSuccess) break;
        k_ct_region_sums<<<blocks(N), CT_THREADS, 0, ctx->stream>>>(H, W, N, c.P, A, R, Cs);
        k_ct_select<<<m, CT_SEL_THREADS, 0, ctx->stream>>>((int)HW, c.P, A, R, Cs, c.emax, c.thr, catphan_size, d_rows);
        ctx->launches += 2;
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(results + k0, d_rows, sizeof(epid_ct_slice) * m, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && scharr) e = cudaMemcpyAsync(scharr + HW * k0, c.E, 8 * N, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && smoothed) e = cudaMemcpyAsync(smoothed + HW * k0, c.S, 8 * N, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && filled) e = cudaMemcpyAsync(filled + HW * k0, c.F, N, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && labels) e = cudaMemcpyAsync(labels + HW * k0, c.P, 4 * N, cudaMemcpyDeviceToHost, ctx->stream);
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

extern "C" int32_t epid_ct_regions(epid_ctx* ctx, const epid_batch* volume, const double* slope, const double* intercept, int32_t slice,
                                   double otsu_disk_radius, const double* gauss_w, int32_t gauss_r, struct epid_ct_region* regions,
                                   int32_t capacity, int32_t* count, double* threshold, double* max_edge) {
    EPID_REQUIRE(count && threshold && max_edge && (regions || capacity == 0), EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(otsu_disk_radius > 0, EPID_ERR_INVALID, "the region table is get_regions of a Slice: otsu_disk_radius must be > 0");
    OtsuDisk disk{};
    bool use_disk = false;
    const int rc0 = ct_check(ctx, volume, slope, intercept, 0, otsu_disk_radius, gauss_w, gauss_r, &disk, &use_disk);
    if (rc0 != EPID_OK) return rc0;
    EPID_REQUIRE(capacity >= 0, EPID_ERR_INVALID, "bad capacity");
    EPID_REQUIRE(slice >= 0 && slice < volume->n, EPID_ERR_INVALID, "slice %d is outside the series of %d", slice, volume->n);
    const int H = volume->h, W = volume->w, HW = H * W;
    const int ext = std::min((int)((double)std::max(H, W) / 100.0), 3) + 1;
    EPID_REQUIRE(ext - 1 < H && ext - 1 < W, EPID_ERR_INVALID, "buffer size may not be greater than labels size");
    EPID_CUDA(cudaSetDevice(ctx->device));

    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
    const size_t o_in = take(sizeof(SliceIn)), o_emax = take(8), o_thr = take(8), o_cnt = take(4);
    const size_t o_E = take(8ull * HW), o_T = take(8ull * HW), o_S = take(8ull * HW), o_P = take(4ull * HW), o_A = take(4ull * HW);
    const size_t o_R = take(8ull * HW), o_C = take(8ull * HW), o_B = take(16ull * HW), o_M = take(24ull * HW);
    const size_t o_rows = take(sizeof(epid_ct_region) * (size_t)std::max(capacity, 1));
    char* d = nullptr;
    EPID_CUDA(cudaMallocAsync((void**)&d, off, ctx->stream));
    CtPlanes c{};
    c.in = (SliceIn*)(d + o_in);
    c.emax = (unsigned long long*)(d + o_emax);
    c.thr = (double*)(d + o_thr);
    c.E = (double*)(d + o_E); c.T = (double*)(d + o_T); c.S = (double*)(d + o_S);
    c.P = (int*)(d + o_P); c.flag = (int*)(d + o_A);
    int* d_cnt = (int*)(d + o_cnt);
    unsigned int* A = (unsigned int*)(d + o_A);
    unsigned long long *R = (unsigned long long*)(d + o_R), *Cs = (unsigned long long*)(d + o_C), *M = (unsigned long long*)(d + o_M);
    int* B = (int*)(d + o_B);
    epid_ct_region* d_rows = (epid_ct_region*)(d + o_rows);
    char* d_ws = nullptr;

    const SliceIn hin{(const char*)volume->dptr + (size_t)slice * HW * dtype_size(volume->dtype), slope[slice], intercept[slice]};
    cudaError_t e = cudaMemcpyAsync(c.in, &hin, sizeof(SliceIn), cudaMemcpyHostToDevice, ctx->stream);
    int rc = EPID_OK;
    unsigned long long emax_bits = 0;
    int n = 0;
    if (e == cudaSuccess) rc = ct_label_chunk(ctx, volume->dtype, c, 1, H, W, true, &disk, false, gauss_w, gauss_r, e);
    if (rc == EPID_OK && e == cudaSuccess) {
        // the flag plane shares A's memory and is done with
        e = cudaMemsetAsync(A, 0, 4ull * HW, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(R, 0, 8ull * HW, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(Cs, 0, 8ull * HW, ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(B, 0x7f, 8ull * HW, ctx->stream);       // min row, min column: large
        if (e == cudaSuccess) e = cudaMemsetAsync(B + 2 * HW, 0, 8ull * HW, ctx->stream);  // max row, max column + 1: 0
        if (e == cudaSuccess) e = cudaMemsetAsync(M, 0, 24ull * HW, ctx->stream);
    }
    if (rc == EPID_OK && e == cudaSuccess) {
        k_ct_region_sums<<<blocks(HW), CT_THREADS, 0, ctx->stream>>>(H, W, HW, c.P, A, R, Cs);
        k_ct_region_bbox<<<blocks(HW), CT_THREADS, 0, ctx->stream>>>(W, HW, c.P, B);
        k_ct_region_moments<<<blocks(HW), CT_THREADS, 0, ctx->stream>>>(W, HW, c.P, B, M);
        k_ct_region_rows<<<1, CT_SEL_THREADS, 0, ctx->stream>>>(HW, c.P, A, R, Cs, B, M, capacity, d_rows, d_cnt);
        ctx->launches += 4;
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(&n, d_cnt, 4, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(threshold, c.thr, 8, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(&emax_bits, c.emax, 8, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        const int nr = std::min(n, capacity);
        if (e == cudaSuccess && nr > 0) e = cudaMemcpy(regions, d_rows, sizeof(epid_ct_region) * nr, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess && nr > 0) {
            // each row's two bitmasks, C and F of its bbox crop, at a word offset of its own
            std::vector<long long> woff(nr);
            long long words = 0;
            for (int k = 0; k < nr; k++) {
                woff[k] = words;
                const long long h = regions[k].bbox[2] - regions[k].bbox[0], w = regions[k].bbox[3] - regions[k].bbox[1];
                words += 2 * h * ((w + 31) / 32);
            }
            const size_t o_words = align256(8 * (size_t)nr);
            e = cudaMallocAsync((void**)&d_ws, o_words + 4 * (size_t)words, ctx->stream);
            long long* d_off = (long long*)d_ws;
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_off, woff.data(), 8 * (size_t)nr, cudaMemcpyHostToDevice, ctx->stream);
            if (e == cudaSuccess) {
                k_ct_region_fill<<<nr, CT_THREADS, 0, ctx->stream>>>(W, c.P, d_rows, d_off, (unsigned int*)(d_ws + o_words));
                ctx->launches += 1;
                e = cudaGetLastError();
            }
            if (e == cudaSuccess) e = cudaMemcpyAsync(regions, d_rows, sizeof(epid_ct_region) * nr, cudaMemcpyDeviceToHost, ctx->stream);
            // woff is read by the stream: wait before it goes out of scope
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        }
    }
    if (d_ws) {
        const cudaError_t ef = cudaFreeAsync(d_ws, ctx->stream);
        if (e == cudaSuccess) e = ef;
    }
    const cudaError_t ef = cudaFreeAsync(d, ctx->stream);
    if (e == cudaSuccess) e = ef;
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (rc != EPID_OK) return rc;
    if (e != cudaSuccess) {
        set_error("epid_ct_regions failed: %s", cudaGetErrorString(e));
        return EPID_ERR_CUDA;
    }
    *count = n;
    std::memcpy(max_edge, &emax_bits, 8);
    return EPID_OK;
}
