// Region statistics on device-resident frames.
//
//   epid_roi_stats          RectangleROI.pixels_flat -> mean / std / min / max (core/roi.py:533-706): the pixels of a (possibly
//                           rotated) rectangle given by its four corners, selected like skimage.draw.polygon does -- integer pixel
//                           coordinates inside the polygon or ON its boundary (skimage's point_in_polygon returns non-zero for
//                           edge and vertex hits), clipped to the image.  skimage is not available in the build container: the
//                           rule is restated from its documentation / source as recalled (parity unpinned at that boundary); for
//                           axis-aligned rectangles with integer corners it reduces to a plain slice.
//   epid_weighted_centroid  WeightedCentroid.calculate (metrics/image.py:959-983): sum(idx * a) / sum(a) along both axes.
//   epid_disk_stats         DiskROI / HighContrastDiskROI (core/roi.py:39-190, 411-478): np.mean / np.std / np.min / np.max /
//                           np.median of arr[skimage.draw.disk((cy, cx), r)], bit for bit, in numpy's own summation orders.
//
// One CTA per (frame, ROI).  Integer dtypes accumulate exact 64-bit sums (count, sum, sum of squares, index-weighted sums); float
// dtypes accumulate in fp64.  std = sqrt(mean(|x - mean|^2)) as numpy defines it, evaluated from the exact moments for integers.
// epid_disk_stats runs one CTA per disk and evaluates numpy's expressions instead (see k_disk_stats).
#include <cmath>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "np_sum.cuh"
#include "roi.cuh"
#include "stats.cuh"

namespace epid {

constexpr int ROI_THREADS = 256;

template <typename T> struct RoiAcc { using type = double; };
template <> struct RoiAcc<uint8_t> { using type = unsigned long long; };
template <> struct RoiAcc<uint16_t> { using type = unsigned long long; };

struct RoiOut { double count, sum, sumsq, mn, mx, varnum; };   // varnum: exact N * S2 - S1^2 for 8 / 16-bit pixels, else -1

template <typename T>
__global__ void __launch_bounds__(ROI_THREADS)
k_roi_stats(const T* __restrict__ data, int H, int W, int nroi, const double* __restrict__ verts, RoiOut* __restrict__ out) {
    using A = typename RoiAcc<T>::type;
    const int fi = blockIdx.y, ri = blockIdx.x;
    const T* f = data + (size_t)fi * H * W;
    const double* v = verts + (size_t)ri * 8;          // (x, y) x 4
    const double vx[4] = {v[0], v[2], v[4], v[6]}, vy[4] = {v[1], v[3], v[5], v[7]};
    const double xmin = fmin(fmin(vx[0], vx[1]), fmin(vx[2], vx[3])), xmax = fmax(fmax(vx[0], vx[1]), fmax(vx[2], vx[3]));
    const double ymin = fmin(fmin(vy[0], vy[1]), fmin(vy[2], vy[3])), ymax = fmax(fmax(vy[0], vy[1]), fmax(vy[2], vy[3]));
    // skimage.draw._polygon: minr = int(max(0, r.min())), maxr = int(ceil(r.max())), clipped to shape - 1
    const int r0 = (int)fmax(0.0, ymin), r1 = min((int)ceil(ymax), H - 1);
    const int c0 = (int)fmax(0.0, xmin), c1 = min((int)ceil(xmax), W - 1);
    const int bh = r1 - r0 + 1, bw = c1 - c0 + 1;
    A s1 = 0, s2 = 0;
    unsigned long long cnt = 0;
    double mn = INFINITY, mx = -INFINITY;
    if (bh > 0 && bw > 0) {
        for (int i = threadIdx.x; i < bh * bw; i += ROI_THREADS) {
            const int r = r0 + i / bw, c = c0 + i % bw;
            if (!point_in_quad(vx, vy, (double)c, (double)r)) continue;
            const T pv = f[(size_t)r * W + c];
            const A a = (A)pv;
            s1 += a;
            s2 += a * a;
            cnt++;
            mn = fmin(mn, (double)pv);
            mx = fmax(mx, (double)pv);
        }
    }
    __shared__ A sh1[ROI_THREADS], sh2[ROI_THREADS];
    __shared__ unsigned long long shc[ROI_THREADS];
    __shared__ double shmn[ROI_THREADS], shmx[ROI_THREADS];
    sh1[threadIdx.x] = s1; sh2[threadIdx.x] = s2; shc[threadIdx.x] = cnt; shmn[threadIdx.x] = mn; shmx[threadIdx.x] = mx;
    __syncthreads();
    for (int s = ROI_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            sh1[threadIdx.x] += sh1[threadIdx.x + s];
            sh2[threadIdx.x] += sh2[threadIdx.x + s];
            shc[threadIdx.x] += shc[threadIdx.x + s];
            shmn[threadIdx.x] = fmin(shmn[threadIdx.x], shmn[threadIdx.x + s]);
            shmx[threadIdx.x] = fmax(shmx[threadIdx.x], shmx[threadIdx.x + s]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        RoiOut o;
        o.count = (double)shc[0];
        o.sum = (double)sh1[0];
        o.sumsq = (double)sh2[0];
        o.mn = shmn[0];
        o.mx = shmx[0];
        o.varnum = -1.0;
        if (!std::is_floating_point<A>::value && shc[0] > 0) {
            // exact population variance numerator N * S2 - S1^2 in 128-bit integer arithmetic -> fp64 once
            const unsigned __int128 n = shc[0];
            const unsigned __int128 num = n * (unsigned __int128)(unsigned long long)sh2[0] -
                                          (unsigned __int128)(unsigned long long)sh1[0] * (unsigned long long)sh1[0];
            o.varnum = (double)num;
        }
        out[(size_t)fi * nroi + ri] = o;
    }
}

template <typename T>
static int do_roi(epid_ctx* ctx, const epid_batch* b, int nroi, const double* d_verts, RoiOut* d_out) {
    k_roi_stats<T><<<dim3(nroi, b->n), ROI_THREADS, 0, ctx->stream>>>((const T*)b->dptr, b->h, b->w, nroi, d_verts, d_out);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

// ---------------------------------------------------------------------------------------- weighted centroid
template <typename T>
__global__ void __launch_bounds__(ROI_THREADS)
k_weighted_centroid(const T* __restrict__ data, int H, int W, double* __restrict__ part) {
    // grid (blocks, n): per-block partial sums of a, x * a, y * a (exact for integer pixels), combined on the host side of the C-ABI
    using A = typename RoiAcc<T>::type;
    const int fi = blockIdx.y;
    const T* f = data + (size_t)fi * H * W;
    A s = 0, sx = 0, sy = 0;
    const size_t per = (size_t)H * W;
    for (size_t i = (size_t)blockIdx.x * ROI_THREADS + threadIdx.x; i < per; i += (size_t)gridDim.x * ROI_THREADS) {
        const A a = (A)f[i];
        const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
        s += a;
        sx += a * (A)x;
        sy += a * (A)y;
    }
    __shared__ A sh[3][ROI_THREADS];
    sh[0][threadIdx.x] = s; sh[1][threadIdx.x] = sx; sh[2][threadIdx.x] = sy;
    __syncthreads();
    for (int k = ROI_THREADS / 2; k > 0; k >>= 1) {
        if (threadIdx.x < k) for (int j = 0; j < 3; j++) sh[j][threadIdx.x] += sh[j][threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x < 3) {
        // integer sums travel as two 32-bit halves in doubles (exact), float sums as they are
        double* o = part + ((size_t)fi * gridDim.x + blockIdx.x) * 6;
        const A v = sh[threadIdx.x][0];
        if (std::is_floating_point<A>::value) { o[2 * threadIdx.x] = (double)v; o[2 * threadIdx.x + 1] = 0.0; }
        else {
            const unsigned long long u = (unsigned long long)v;
            o[2 * threadIdx.x] = (double)(u >> 32);
            o[2 * threadIdx.x + 1] = (double)(u & 0xffffffffull);
        }
    }
}

constexpr int WC_BLOCKS = 64;
template <typename T>
static int do_wc(epid_ctx* ctx, const epid_batch* b, double* d_part) {
    k_weighted_centroid<T><<<dim3(WC_BLOCKS, b->n), ROI_THREADS, 0, ctx->stream>>>((const T*)b->dptr, b->h, b->w, d_part);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}


// ---------------------------------------------------------------------------------------------------- disk statistics
// The pixels of skimage.draw.disk((cy, cx), r) without `shape` (ellipse with rotation 0): the bounding box ceil(c - r) .. floor(c + r),
// float offsets (i - (cy - r0)) / r and (j - (cx - c0)) / r from the centre, membership a*a + b*b < 1 (built with -fmad=false, so it
// rounds as numpy does), raster order; arr[rr, cc] wraps negative indices.  The member columns of one row are one run (the test is
// monotone in |j - cx| after rounding), so each row is (first column, length) and a prefix over the lengths maps a raster index to its
// pixel: the pairwise sums read the frame through that map and nothing is gathered.
//
// numpy's expressions, per dtype (numpy/_core/_methods.py _mean / _var, lib/_function_base_impl.py median):
//   mean    integers: float64 pairwise sums over the casting buffer's chunks of 8192 values, added in sequence from 0, / n;
//           float32: a float32 pairwise sum, float32(float64(sum) / n); float64: 0 + one pairwise sum, / n.
//   std     d = x - mean in the mean's type, d * d, 0 + one pairwise sum of the squares (no cast, no chunks), var as the mean is
//           formed, sqrt in that type.
//   median  the one or two middle order statistics (radix select over order-preserving keys, 8 bits a pass), then np.mean of them;
//           any NaN makes it NaN (numpy's _median_nancheck), as it does min and max.
constexpr int DISK_THREADS = 256, DISK_LOG_THREADS = 8, DISK_WARPS = DISK_THREADS / 32;
constexpr int DISK_MAX_ROWS = 16384;          // rows (and columns) of a disk's bounding box: the row table lives in shared memory
constexpr long long NP_CAST_BUFFER = 8192;    // numpy's ufunc buffer: a cast reduction sums in chunks of this many values

template <typename T> struct DiskTraits {      // unsigned integers of 8 / 16 bits
    using Key = uint32_t; using Acc = double;
    static constexpr bool integral = true;
    __device__ static Key key(T v) { return v; }
    __device__ static T value(Key k) { return (T)k; }
};
template <> struct DiskTraits<int16_t> {
    using Key = uint32_t; using Acc = double;
    static constexpr bool integral = true;
    __device__ static Key key(int16_t v) { return (uint32_t)(uint16_t)v ^ 0x8000u; }
    __device__ static int16_t value(Key k) { return (int16_t)(uint16_t)(k ^ 0x8000u); }
};
template <> struct DiskTraits<int32_t> {
    using Key = uint32_t; using Acc = double;
    static constexpr bool integral = true;
    __device__ static Key key(int32_t v) { return (uint32_t)v ^ 0x80000000u; }
    __device__ static int32_t value(Key k) { return (int32_t)(k ^ 0x80000000u); }
};
template <> struct DiskTraits<long long> {
    using Key = unsigned long long; using Acc = double;
    static constexpr bool integral = true;
    __device__ static Key key(long long v) { return (unsigned long long)v ^ 0x8000000000000000ull; }
    __device__ static long long value(Key k) { return (long long)(k ^ 0x8000000000000000ull); }
};
template <> struct DiskTraits<float> {
    using Key = uint32_t; using Acc = float;
    static constexpr bool integral = false;
    __device__ static Key key(float v) { const uint32_t u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : u | 0x80000000u; }
    __device__ static float value(Key k) { return __uint_as_float((k & 0x80000000u) ? k & 0x7fffffffu : ~k); }
};
template <> struct DiskTraits<double> {
    using Key = unsigned long long; using Acc = double;
    static constexpr bool integral = false;
    __device__ static Key key(double v) {
        const unsigned long long u = (unsigned long long)__double_as_longlong(v);
        return (u & 0x8000000000000000ull) ? ~u : u | 0x8000000000000000ull;
    }
    __device__ static double value(Key k) {
        return __longlong_as_double((long long)((k & 0x8000000000000000ull) ? k & 0x7fffffffffffffffull : ~k));
    }
};

struct DiskOut { double count, mean, std, mn, mx, median; };   // count < 0: a member pixel lies beyond the frame (numpy's IndexError)

// member j of row i of a disk's row table, negative indices wrapped as numpy's fancy indexing does
template <typename T> struct DiskPixel {
    const T* f;
    const int* lo;
    long long r0, c0;
    int H, W;
    __device__ T operator()(int i, long long j) const {
        long long r = r0 + i, c = c0 + lo[i] + j;
        if (r < 0) r += H;
        if (c < 0) c += W;
        return f[r * W + c];
    }
};

// The row table of one disk in shared memory: lo[i] is row i's first member column and pre[i] the members before row i (pre[bh] = n),
// with numpy's bounds check of every member index.  Returns n, or -1 when a member lies beyond the frame (numpy's IndexError).  Every
// thread of the CTA calls it, once per CTA; kept out of line, which keeps k_disk_percentiles from spilling.
__device__ __noinline__ long long disk_rows_table(const DiskBox& box, double sr, double sc, double R, int H, int W, int* lo, int* pre) {
    __shared__ long long part[DISK_THREADS];
    __shared__ int s_bad;
    const int tid = threadIdx.x;
    const int bh = (int)box.bh, bw = (int)box.bw;
    if (tid == 0) { s_bad = 0; pre[0] = 0; }
    __syncthreads();

    // each row's run of member columns, and numpy's bounds check of every member index
    for (int i = tid; i < bh; i += DISK_THREADS) {
        const double a = ((double)i - sr) / R;
        const double aa = a * a;
        int first = -1, last = -2;
        for (int j = 0; j < bw; j++) {
            const double b = ((double)j - sc) / R;
            if (aa + b * b < 1.0) { if (first < 0) first = j; last = j; }
        }
        const int len = last - first + 1;
        lo[i] = first < 0 ? 0 : first;
        pre[i + 1] = len;
        if (len > 0) {
            const long long r = box.r0 + i, c_first = box.c0 + first, c_last = box.c0 + last;
            if (r < -H || r >= H || c_first < -W || c_last >= W) s_bad = 1;
        }
    }
    __syncthreads();
    // prefix over the run lengths: a serial chunk per thread, one serial pass over the chunk totals
    const int chunk = (bh + DISK_THREADS - 1) / DISK_THREADS;
    const int i0 = min(bh, tid * chunk), i1 = min(bh, i0 + chunk);
    long long run = 0;
    for (int i = i0; i < i1; i++) run += pre[i + 1];
    part[tid] = run;
    __syncthreads();
    if (tid == 0) {
        long long acc = 0;
        for (int t = 0; t < DISK_THREADS; t++) { const long long v = part[t]; part[t] = acc; acc += v; }
    }
    __syncthreads();
    run = part[tid];
    for (int i = i0; i < i1; i++) { run += pre[i + 1]; pre[i + 1] = (int)run; }
    __syncthreads();
    if (s_bad) return -1;
    return bh > 0 ? pre[bh] : 0;
}

// The order statistics of ranks k and, with `next`, k + 1 (0-based) of the disk's pixels in DiskTraits' key order, by radix select:
// 8 bits a pass, each pass a 256-bin shared histogram of the keys that match the digits chosen so far, so no pixel is buffered.  Rank
// k + 1 is rank k's key again while that key's count covers it, else the smallest key above it (one more pass).  Every thread of
// the CTA calls it with the same arguments and receives both values (b = a without `next`).
template <typename T>
__device__ __forceinline__ void disk_select(const DiskPixel<T>& pixel, const int* pre, int bh, long long k, bool next, T& a, T& b) {
    using Tr = DiskTraits<T>;
    using K = typename Tr::Key;
    __shared__ unsigned int hist[256];
    __shared__ int s_digit;
    __shared__ long long s_k, s_eq;
    __shared__ unsigned long long s_next;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    K prefix = 0, mask = 0;
    for (int shift = 8 * ((int)sizeof(T) - 1); shift >= 0; shift -= 8) {
        for (int d = tid; d < 256; d += DISK_THREADS) hist[d] = 0;
        __syncthreads();
        for (int i = warp; i < bh; i += DISK_WARPS) {
            const int len = pre[i + 1] - pre[i];
            for (int j = lane; j < len; j += 32) {
                const K key = Tr::key(pixel(i, j));
                if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
            }
        }
        __syncthreads();
        if (tid == 0) {
            long long acc = 0;
            int dg = 0;
            for (; dg < 255; dg++) {
                if (k < acc + (long long)hist[dg]) break;
                acc += hist[dg];
            }
            s_digit = dg;
            s_k = k - acc;
            s_eq = hist[dg];
        }
        __syncthreads();
        prefix |= (K)s_digit << shift;
        mask |= (K)255u << shift;
        k = s_k;
    }
    a = b = Tr::value(prefix);
    if (next && k + 1 >= s_eq) {                     // the next order statistic is the smallest key above a's
        if (tid == 0) s_next = ~0ull;
        __syncthreads();
        unsigned long long best = ~0ull;
        for (int i = warp; i < bh; i += DISK_WARPS) {
            const int len = pre[i + 1] - pre[i];
            for (int j = lane; j < len; j += 32) {
                const K key = Tr::key(pixel(i, j));
                if (key > prefix && (unsigned long long)key < best) best = key;
            }
        }
        atomicMin(&s_next, best);
        __syncthreads();
        b = Tr::value((K)s_next);
    }
}

// CTAs an SM that k_disk_stats asks of ptxas: the occupancy of the kernel before its select moved into disk_select, 3 for float64 and
// uint8 (at most 85 registers), 4 for the others (64).  The kernel is latency-bound; without a bound ptxas takes 80 to 96 registers,
// and at 80 (3 CTAs) uint16 measured 7 % slower than at 64.  At 64 the 16- to 64-bit integers reload 80 spilled bytes.
template <typename T> constexpr int DISK_STATS_MIN_CTAS = std::is_same<T, double>::value || std::is_same<T, uint8_t>::value ? 3 : 4;

template <typename T>
__global__ void __launch_bounds__(DISK_THREADS, DISK_STATS_MIN_CTAS<T>)
k_disk_stats(const T* __restrict__ data, int H, int W, const double* __restrict__ disks, DiskOut* __restrict__ out) {
    using Tr = DiskTraits<T>;
    using A = typename Tr::Acc;
    extern __shared__ int disk_rows[];              // lo[bh]: first member column; pre[bh + 1]: members before each row
    __shared__ A slots[DISK_THREADS];
    __shared__ double wmn[DISK_WARPS], wmx[DISK_WARPS];
    __shared__ int s_nan;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double* dk = disks + (size_t)blockIdx.x * 4;
    const T* f = data + (size_t)(long long)dk[0] * H * W;
    const double cy = dk[1], cx = dk[2], R = dk[3];
    const DiskBox box = disk_box(cy, cx, R);
    const int bh = (int)box.bh;
    int* lo = disk_rows;
    int* pre = disk_rows + bh;
    if (tid == 0) s_nan = 0;
    const long long n = disk_rows_table(box, cy - (double)box.r0, cx - (double)box.c0, R, H, W, lo, pre);   // skimage's `shifted`
    DiskOut o;
    o.count = (double)n;
    o.mean = o.std = o.mn = o.mx = o.median = NAN;
    if (n <= 0) {
        if (tid == 0) out[blockIdx.x] = o;
        return;
    }
    const DiskPixel<T> pixel{f, lo, box.r0, box.c0, H, W};
    auto at = [&](long long k) -> T {                // raster index k -> its pixel: the last row i with pre[i] <= k
        int a = 0, b = bh - 1;
        while (a < b) {
            const int m = (a + b + 1) >> 1;
            if (pre[m] <= k) a = m; else b = m - 1;
        }
        return pixel(a, k - pre[a]);
    };

    // min / max / NaN, in any order
    double mn = INFINITY, mx = -INFINITY;
    int has_nan = 0;
    for (int i = warp; i < bh; i += DISK_WARPS) {
        const int len = pre[i + 1] - pre[i];
        for (int j = lane; j < len; j += 32) {
            const double v = (double)pixel(i, j);
            if (v != v) has_nan = 1;
            mn = fmin(mn, v);
            mx = fmax(mx, v);
        }
    }
    for (int off = 16; off > 0; off >>= 1) {
        mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    if (lane == 0) { wmn[warp] = mn; wmx[warp] = mx; }
    if (has_nan) s_nan = 1;
    __syncthreads();
    const bool any_nan = s_nan != 0;
    if (!any_nan) {
        mn = wmn[0];
        mx = wmx[0];
        for (int w = 1; w < DISK_WARPS; w++) { mn = fmin(mn, wmn[w]); mx = fmax(mx, wmx[w]); }
        o.mn = mn;
        o.mx = mx;
    }

    // np.mean
    A sum = 0.0;
    const long long step = Tr::integral ? NP_CAST_BUFFER : n;
    for (long long c0 = 0; c0 < n; c0 += step) {
        const long long len = min(step, n - c0);
        sum = sum + np::block_pw([&](long long k) -> A { return (A)at(c0 + k); }, len, DISK_LOG_THREADS, slots);
    }
    const A mean = (A)((double)sum / (double)n);
    o.mean = (double)mean;
    // np.std
    const A ss = (A)0.0 + np::block_pw([&](long long k) -> A { const A d = (A)at(k) - mean; return d * d; }, n, DISK_LOG_THREADS, slots);
    const A var = (A)((double)ss / (double)n);
    o.std = (double)sqrt(var);

    // np.median: rank (n - 1) / 2, and for even n the next order statistic
    if (!any_nan) {
        T a, b;
        disk_select<T>(pixel, pre, bh, n % 2 ? n / 2 : n / 2 - 1, n % 2 == 0, a, b);
        if (n % 2) o.median = (double)(A)((double)((A)0.0 + ((A)-0.0 + (A)a)) / 1.0);
        else o.median = (double)(A)((double)((A)0.0 + (((A)-0.0 + (A)a) + (A)b)) / 2.0);
    }
    if (tid == 0) out[blockIdx.x] = o;
}

// np.percentile(arr[disk], q) (method "linear") of one disk per CTA for nq percentiles.  numpy plans and interpolates in the result's
// type: float32 for a float32 array (q / float32(100), the virtual index and the lerp all in float32), float64 for every other dtype.
// An integer array forms b - a in its own type, wrapping, before the lerp.  Each distinct rank the plans name is selected once, and a
// rank k followed by k + 1 in one select.  Any NaN pixel gives NaN (np.percentile returns the NaN that sorts last).
constexpr int DISK_MAX_Q = 16;
template <typename T> using PctType = typename std::conditional<std::is_same<T, float>::value, float, double>::type;

template <typename T>
__global__ void __launch_bounds__(DISK_THREADS)
k_disk_percentiles(const T* __restrict__ data, int H, int W, const double* __restrict__ disks, int nq, const double* __restrict__ q_percent,
                   double* __restrict__ out, long long* __restrict__ count) {
    using F = PctType<T>;
    extern __shared__ int disk_rows[];
    __shared__ long long s_rank[2 * DISK_MAX_Q];    // the distinct ranks the plans read, ascending
    __shared__ T s_val[2 * DISK_MAX_Q];
    __shared__ int s_nr, s_ia[DISK_MAX_Q], s_ib[DISK_MAX_Q];   // each q's two ranks, as indices into s_rank
    __shared__ F s_t[DISK_MAX_Q];                   // and its weight
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double* dk = disks + (size_t)blockIdx.x * 4;
    const T* f = data + (size_t)(long long)dk[0] * H * W;
    const double cy = dk[1], cx = dk[2], R = dk[3];
    const DiskBox box = disk_box(cy, cx, R);
    const int bh = (int)box.bh;
    int* lo = disk_rows;
    int* pre = disk_rows + bh;
    const long long n = disk_rows_table(box, cy - (double)box.r0, cx - (double)box.c0, R, H, W, lo, pre);
    if (tid == 0) count[blockIdx.x] = n;
    double* o = out + (size_t)blockIdx.x * nq;
    const DiskPixel<T> pixel{f, lo, box.r0, box.c0, H, W};
    bool nan = n <= 0;
    if constexpr (!std::is_integral<T>::value) {
        if (!nan) for (int i = warp; i < bh; i += DISK_WARPS) {
            const int len = pre[i + 1] - pre[i];
            for (int j = lane; j < len; j += 32) { const T v = pixel(i, j); if (v != v) nan = true; }
        }
    }
    if (__syncthreads_or(nan)) {
        for (int k = tid; k < nq; k += DISK_THREADS) o[k] = NAN;
        return;
    }
    if (tid == 0) {
        int nr = 0;
        for (int k = 0; k < nq; k++) {
            const F q = (F)q_percent[k];
            const PctPlanOf<F> p = pct_plan((int)n, q);
            for (int u = 0; u < 2; u++) {               // insert prev, then next, into the ascending list of distinct ranks
                const long long r = u ? p.next : p.prev;
                int at = nr;
                while (at > 0 && s_rank[at - 1] > r) at--;
                if (at > 0 && s_rank[at - 1] == r) continue;
                for (int m = nr; m > at; m--) s_rank[m] = s_rank[m - 1];
                s_rank[at] = r;
                nr++;
            }
            // numpy's weight is the virtual index less the previous index, which is -1 past the end (_get_indexes, _get_gamma); it
            // differs from pct_plan's gamma only there and at q = -0, where it changes the sign of a zero result
            const F vi = (F)(n - 1) * (q / (F)100.0);
            s_t[k] = (F)((double)vi - (vi >= (F)(n - 1) ? -1.0 : (double)p.prev));
            s_ia[k] = p.prev;                           // a rank for now; an index into s_rank below
            s_ib[k] = p.next;
        }
        for (int k = 0; k < nq; k++) {
            int ia = 0, ib = 0;
            while (s_rank[ia] != s_ia[k]) ia++;
            while (s_rank[ib] != s_ib[k]) ib++;
            s_ia[k] = ia;
            s_ib[k] = ib;
        }
        s_nr = nr;
    }
    __syncthreads();
    for (int r = 0; r < s_nr;) {
        const bool next = r + 1 < s_nr && s_rank[r + 1] == s_rank[r] + 1;
        T a, b;
        disk_select<T>(pixel, pre, bh, s_rank[r], next, a, b);
        if (tid == 0) { s_val[r] = a; s_val[r + next] = b; }
        r += next ? 2 : 1;
    }
    __syncthreads();
    for (int k = tid; k < nq; k += DISK_THREADS) {
        const T a = s_val[s_ia[k]], b = s_val[s_ib[k]];
        const F t = s_t[k];
        F d = (F)b - (F)a;
        if constexpr (std::is_integral<T>::value) {
            using U = typename std::make_unsigned<T>::type;
            d = (F)(T)(U)((U)b - (U)a);
        }
        o[k] = (double)np_lerp_d((F)a, (F)b, d, t);
    }
}

template <typename T>
static int do_disk(epid_ctx* ctx, const epid_batch* b, int ndisk, const double* d_disks, DiskOut* d_out, size_t smem) {
    if (smem > 48 * 1024) EPID_SMEM_OPT_IN(ctx, k_disk_stats<T>, smem);
    k_disk_stats<T><<<ndisk, DISK_THREADS, smem, ctx->stream>>>((const T*)b->dptr, b->h, b->w, d_disks, d_out);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

template <typename T>
static int do_disk_pct(epid_ctx* ctx, const epid_batch* b, int ndisk, const double* d_disks, int nq, const double* d_q, double* d_out,
                       long long* d_count, size_t smem) {
    if (smem > 48 * 1024) EPID_SMEM_OPT_IN(ctx, k_disk_percentiles<T>, smem);
    k_disk_percentiles<T><<<ndisk, DISK_THREADS, smem, ctx->stream>>>((const T*)b->dptr, b->h, b->w, d_disks, nq, d_q, d_out, d_count);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace epid

using namespace epid;

#define EPID_DISPATCH_ROI(dt, FN, ...)                                              \
    switch (dt) {                                                                   \
        case EPID_U8: rc = FN<uint8_t>(__VA_ARGS__); break;                         \
        case EPID_U16: rc = FN<uint16_t>(__VA_ARGS__); break;                       \
        case EPID_I16: rc = FN<int16_t>(__VA_ARGS__); break;                        \
        case EPID_I32: rc = FN<int32_t>(__VA_ARGS__); break;                        \
        case EPID_I64: rc = FN<long long>(__VA_ARGS__); break;                      \
        case EPID_F32: rc = FN<float>(__VA_ARGS__); break;                          \
        case EPID_F64: rc = FN<double>(__VA_ARGS__); break;                         \
        default: set_error("unknown dtype %d", dt); rc = EPID_ERR_INVALID;          \
    }

extern "C" int32_t epid_roi_stats(epid_ctx* ctx, const epid_batch* b, int32_t nroi, const double* verts_xy, double* count, double* mean,
                                  double* std, double* mn, double* mx) {
    EPID_REQUIRE(ctx && b && verts_xy && nroi > 0 && nroi <= 4096, EPID_ERR_INVALID, "bad argument");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t nv = sizeof(double) * 8 * nroi, no = sizeof(RoiOut) * (size_t)nroi * b->n;
    int rc = ensure_scratch(ctx, nv + no + 512);
    if (rc != EPID_OK) return rc;
    double* d_verts = (double*)ctx->scratch;
    RoiOut* d_out = (RoiOut*)((char*)ctx->scratch + align256(nv));
    EPID_CUDA(cudaMemcpyAsync(d_verts, verts_xy, nv, cudaMemcpyHostToDevice, ctx->stream));
    EPID_DISPATCH_ROI(b->dtype, do_roi, ctx, b, nroi, d_verts, d_out);
    if (rc != EPID_OK) return rc;
    std::vector<RoiOut> h((size_t)nroi * b->n);
    EPID_CUDA(cudaMemcpyAsync(h.data(), d_out, no, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < h.size(); i++) {
        const RoiOut& o = h[i];
        const double n = o.count;
        if (count) count[i] = n;
        const double m = n > 0 ? o.sum / n : NAN;
        if (mean) mean[i] = m;
        if (std) {
            if (!(n > 0)) std[i] = NAN;
            else if (o.varnum >= 0) std[i] = sqrt(o.varnum) / n;   // exact numerator
            else { const double var = o.sumsq / n - m * m; std[i] = var > 0 ? sqrt(var) : 0.0; }
        }
        if (mn) mn[i] = n > 0 ? o.mn : NAN;
        if (mx) mx[i] = n > 0 ? o.mx : NAN;
    }
    return EPID_OK;
}

extern "C" int32_t epid_weighted_centroid(epid_ctx* ctx, const epid_batch* b, double* cx, double* cy, double* total) {
    EPID_REQUIRE(ctx && b && cx && cy, EPID_ERR_INVALID, "NULL argument");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t np = sizeof(double) * 6 * WC_BLOCKS * (size_t)b->n;
    int rc = ensure_scratch(ctx, np + 256);
    if (rc != EPID_OK) return rc;
    double* d_part = (double*)ctx->scratch;
    EPID_DISPATCH_ROI(b->dtype, do_wc, ctx, b, d_part);
    if (rc != EPID_OK) return rc;
    std::vector<double> h((size_t)6 * WC_BLOCKS * b->n);
    EPID_CUDA(cudaMemcpyAsync(h.data(), d_part, np, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    const bool integral = b->dtype == EPID_U8 || b->dtype == EPID_U16;
    for (int fi = 0; fi < b->n; fi++) {
        if (integral) {      // exact 128-bit totals of the 64 block partials, one fp64 division at the end like numpy's
            unsigned __int128 t[3] = {0, 0, 0};
            for (int k = 0; k < WC_BLOCKS; k++) {
                const double* o = &h[((size_t)fi * WC_BLOCKS + k) * 6];
                for (int j = 0; j < 3; j++) t[j] += ((unsigned __int128)(unsigned long long)o[2 * j] << 32) + (unsigned long long)o[2 * j + 1];
            }
            const double s = (double)t[0];
            if (total) total[fi] = s;
            cx[fi] = (double)t[1] / s;
            cy[fi] = (double)t[2] / s;
        } else {
            double t[3] = {0, 0, 0};
            for (int k = 0; k < WC_BLOCKS; k++) for (int j = 0; j < 3; j++) t[j] += h[((size_t)fi * WC_BLOCKS + k) * 6 + 2 * j];
            if (total) total[fi] = t[0];
            cx[fi] = t[1] / t[0];
            cy[fi] = t[2] / t[0];
        }
    }
    return EPID_OK;
}

// the disk rows' checks shared by the disk entry points; *max_rows: the most bounding-box rows of any disk
static int check_disks(const epid_batch* b, int ndisk, const double* disks, long long* max_rows) {
    *max_rows = 0;
    for (int i = 0; i < ndisk; i++) {
        const double* d = disks + (size_t)i * 4;
        EPID_REQUIRE(d[0] >= 0 && d[0] < b->n && d[0] == floor(d[0]), EPID_ERR_INVALID, "disk %d: frame index %g outside the batch of %d",
                     i, d[0], b->n);
        EPID_REQUIRE(isfinite(d[1]) && isfinite(d[2]) && isfinite(d[3]), EPID_ERR_INVALID, "disk %d: non-finite geometry", i);
        EPID_REQUIRE(fabs(d[1]) < 1e9 && fabs(d[2]) < 1e9 && fabs(d[3]) < 1e9, EPID_ERR_UNSUPPORTED, "disk %d: geometry beyond 1e9 px", i);
        const DiskBox bx = disk_box(d[1], d[2], d[3]);
        EPID_REQUIRE(bx.bh <= DISK_MAX_ROWS && bx.bw <= DISK_MAX_ROWS, EPID_ERR_UNSUPPORTED,
                     "disk %d: a %lld x %lld bounding box exceeds %d rows or columns", i, bx.bh, bx.bw, DISK_MAX_ROWS);
        if (bx.bh > *max_rows) *max_rows = bx.bh;
    }
    return EPID_OK;
}

extern "C" int32_t epid_disk_stats(epid_ctx* ctx, const epid_batch* b, int32_t ndisk, const double* disks, double* count, double* mean,
                                   double* std, double* mn, double* mx, double* median) {
    EPID_REQUIRE(ctx && b && (disks || ndisk == 0) && ndisk >= 0, EPID_ERR_INVALID, "bad argument");
    if (ndisk == 0) return EPID_OK;
    long long max_rows = 0;
    int rc = check_disks(b, ndisk, disks, &max_rows);
    if (rc != EPID_OK) return rc;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t nd = sizeof(double) * 4 * ndisk, no = sizeof(DiskOut) * (size_t)ndisk;
    rc = ensure_scratch(ctx, nd + no + 512);
    if (rc != EPID_OK) return rc;
    double* d_disks = (double*)ctx->scratch;
    DiskOut* d_out = (DiskOut*)((char*)ctx->scratch + align256(nd));
    EPID_CUDA(cudaMemcpyAsync(d_disks, disks, nd, cudaMemcpyHostToDevice, ctx->stream));
    const size_t smem = sizeof(int) * (size_t)(2 * max_rows + 1);
    EPID_DISPATCH_ROI(b->dtype, do_disk, ctx, b, ndisk, d_disks, d_out, smem);
    if (rc != EPID_OK) return rc;
    std::vector<DiskOut> h(ndisk);
    EPID_CUDA(cudaMemcpyAsync(h.data(), d_out, no, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < ndisk; i++) {
        const DiskOut& o = h[i];
        EPID_REQUIRE(o.count >= 0, EPID_ERR_INVALID, "disk %d: a member pixel lies beyond the %d x %d frame", i, b->h, b->w);
        if (count) count[i] = o.count;
        if (mean) mean[i] = o.mean;
        if (std) std[i] = o.std;
        if (mn) mn[i] = o.mn;
        if (mx) mx[i] = o.mx;
        if (median) median[i] = o.median;
    }
    return EPID_OK;
}

extern "C" int32_t epid_disk_percentiles(epid_ctx* ctx, const epid_batch* b, int32_t ndisk, const double* disks, int32_t nq,
                                         const double* q_percent, double* out) {
    EPID_REQUIRE(ctx && b && (disks || ndisk == 0) && ndisk >= 0, EPID_ERR_INVALID, "bad argument");
    EPID_REQUIRE(nq >= 1 && nq <= DISK_MAX_Q && q_percent && (out || ndisk == 0), EPID_ERR_INVALID, "%d percentiles: 1 to %d are supported",
                 nq, DISK_MAX_Q);
    for (int k = 0; k < nq; k++) {             // np.percentile checks q / 100 in the type it plans in (float32 for a float32 batch)
        const double q = b->dtype == EPID_F32 ? (double)((float)q_percent[k] / 100.0f) : q_percent[k] / 100.0;
        EPID_REQUIRE(q >= 0.0 && q <= 1.0, EPID_ERR_INVALID, "Percentiles must be in the range [0, 100]");
    }
    if (ndisk == 0) return EPID_OK;
    long long max_rows = 0;
    int rc = check_disks(b, ndisk, disks, &max_rows);
    if (rc != EPID_OK) return rc;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t nd = sizeof(double) * 4 * ndisk, nqb = sizeof(double) * nq, no = sizeof(double) * (size_t)ndisk * nq,
                 nc = sizeof(long long) * (size_t)ndisk;
    rc = ensure_scratch(ctx, align256(nd) + align256(nqb) + align256(no) + nc + 256);
    if (rc != EPID_OK) return rc;
    double* d_disks = (double*)ctx->scratch;
    double* d_q = (double*)((char*)d_disks + align256(nd));
    double* d_out = (double*)((char*)d_q + align256(nqb));
    long long* d_count = (long long*)((char*)d_out + align256(no));
    EPID_CUDA(cudaMemcpyAsync(d_disks, disks, nd, cudaMemcpyHostToDevice, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(d_q, q_percent, nqb, cudaMemcpyHostToDevice, ctx->stream));
    const size_t smem = sizeof(int) * (size_t)(2 * max_rows + 1);
    EPID_DISPATCH_ROI(b->dtype, do_disk_pct, ctx, b, ndisk, d_disks, nq, d_q, d_out, d_count, smem);
    if (rc != EPID_OK) return rc;
    std::vector<long long> cnt(ndisk);
    EPID_CUDA(cudaMemcpyAsync(out, d_out, no, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(cnt.data(), d_count, nc, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < ndisk; i++)
        EPID_REQUIRE(cnt[i] >= 0, EPID_ERR_INVALID, "disk %d: a member pixel lies beyond the %d x %d frame", i, b->h, b->w);
    return EPID_OK;
}
