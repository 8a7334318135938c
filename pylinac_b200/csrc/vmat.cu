// VMAT (DRGS / DRMLC) and DLG on device-resident frames.
//
//   epid_vmat_analyze   VMATBase.__init__ / analyze + VMATLinearBase (vmat.py:249-275, 309-346, 408-436, 721-841): n independent image
//                       pairs.  Four launches per batch, no host round trip in between:
//     k_vmat_front      one read of both frames: min / max / total and exact integer column sums (the only HBM-proportional work;
//                       algorithmic bytes = 2 x H x W x 2 per pair)
//     k_vmat_profile    CTA per pair: ground() / check_inversion() of both images as an affine map v -> sign * v + offset of the raw
//                       pixels (uint16 modular arithmetic of the reference never wraps: every intermediate stays inside [min, max]),
//                       the column-mean FWXMProfile of _roi_profiles (ground, beam-centre normalisation, stretch, 90th percentile
//                       normalisation, field_values at 80 %), image identification, field centre
//     k_vmat_segments   CTA per (segment, pair): mean / std of DMLC / open over the pixels RectangleROI.pixels_flat selects
//                       (skimage.draw.polygon rule, roi.cuh); the ratio image itself is never written
//     k_vmat_finalize   R_dev, pass / fail, aggregates
//   epid_divide         the ratio image as a float64 batch (DRCS needs it for CircleProfile / rotated segments)
//   epid_dlg_analyze    DLG.analyze (dlg.py:32-86, 112-127)
//
// All 1-D arithmetic is fp64 in the reference's operation order (-fmad=false); sums of uint16 pixels are exact integers.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "peaks.cuh"
#include "roi.cuh"
#include "profile1d.cuh"

namespace epid {

constexpr int VM_ROWS = 64;          // rows per CTA of the front kernel
constexpr int VM_THREADS = 256;

struct VmAcc { unsigned int mn, mx; unsigned long long sum; };

// ------------------------------------------------------------------------------------------------ front: one read of both frames
__global__ void k_vmat_init(VmAcc* acc, unsigned long long* colsum, size_t nf, size_t ncol) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nf) { acc[i].mn = 0xffffffffu; acc[i].mx = 0; acc[i].sum = 0; }
    for (size_t k = i; k < ncol; k += (size_t)gridDim.x * blockDim.x) colsum[k] = 0;
}

__global__ void k_vmat_front(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b, int n, int H, int W, VmAcc* acc,
                             unsigned long long* colsum) {
    const int f = blockIdx.y;
    const uint16_t* img = f < n ? a + (size_t)f * H * W : b + (size_t)(f - n) * H * W;
    const int r0 = blockIdx.x * VM_ROWS, r1 = min(H, r0 + VM_ROWS);
    unsigned int mn = 0xffffu, mx = 0;
    unsigned long long tot = 0;
    if ((W & 1) == 0) {      // two columns per thread, 32-bit loads (frames are 4-byte aligned when W is even)
        const uint32_t* img2 = reinterpret_cast<const uint32_t*>(img);
        const int W2 = W >> 1;
        for (int c = threadIdx.x; c < W2; c += blockDim.x) {
            unsigned int s0 = 0, s1 = 0;
            int r = r0;
            for (; r + 8 <= r1; r += 8) {
                uint32_t v[8];
#pragma unroll
                for (int k = 0; k < 8; k++) v[k] = __ldg(img2 + (size_t)(r + k) * W2 + c);
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const unsigned int lo = v[k] & 0xffffu, hi = v[k] >> 16;
                    s0 += lo; s1 += hi;
                    mn = min(mn, min(lo, hi)); mx = max(mx, max(lo, hi));
                }
            }
            for (; r < r1; r++) {
                const uint32_t v = __ldg(img2 + (size_t)r * W2 + c);
                const unsigned int lo = v & 0xffffu, hi = v >> 16;
                s0 += lo; s1 += hi;
                mn = min(mn, min(lo, hi)); mx = max(mx, max(lo, hi));
            }
            atomicAdd(&colsum[(size_t)f * W + 2 * c], (unsigned long long)s0);
            atomicAdd(&colsum[(size_t)f * W + 2 * c + 1], (unsigned long long)s1);
            tot += (unsigned long long)s0 + s1;
        }
    } else {
        for (int c = threadIdx.x; c < W; c += blockDim.x) {
            unsigned int s = 0;
            for (int r = r0; r < r1; r++) {
                const unsigned int v = img[(size_t)r * W + c];
                s += v; mn = min(mn, v); mx = max(mx, v);
            }
            atomicAdd(&colsum[(size_t)f * W + c], (unsigned long long)s);
            tot += s;
        }
    }
    mn = warp_min(mn); mx = warp_max(mx); tot = warp_sum(tot);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&acc[f].mn, mn);
        atomicMax(&acc[f].mx, mx);
        atomicAdd(&acc[f].sum, tot);
    }
}

// W % 8 == 0: 16-byte loads, 8 columns per thread, RG row groups per CTA (blockDim = (W / 8) * RG); four independent loads per thread
// in flight.  Column sums of the row groups are combined in shared memory before the global atomics.
__global__ void k_vmat_front_v16(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b, int n, int H, int W, int RG, VmAcc* acc,
                                 unsigned long long* colsum) {
    extern __shared__ unsigned int s_col[];      // [RG][W]
    const int f = blockIdx.y;
    const uint16_t* img = f < n ? a + (size_t)f * H * W : b + (size_t)(f - n) * H * W;
    const int nvec = W >> 3;
    const int j = threadIdx.x % nvec, g = threadIdx.x / nvec;
    const int r0 = blockIdx.x * VM_ROWS, r1 = min(H, r0 + VM_ROWS);
    const uint4* base = reinterpret_cast<const uint4*>(img) + j;
    unsigned int cs[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    unsigned int mn2 = 0xffffffffu, mx2 = 0;
    auto eat = [&](const uint4 q) {
        const unsigned int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int t = 0; t < 4; t++) {
            cs[2 * t] += w[t] & 0xffffu;
            cs[2 * t + 1] += w[t] >> 16;
            mn2 = __vminu2(mn2, w[t]);
            mx2 = __vmaxu2(mx2, w[t]);
        }
    };
    int r = r0 + g;
    for (; r + 3 * RG < r1; r += 4 * RG) {
        const uint4 q0 = ldg_stream16(base + (size_t)r * nvec), q1 = ldg_stream16(base + (size_t)(r + RG) * nvec);
        const uint4 q2 = ldg_stream16(base + (size_t)(r + 2 * RG) * nvec), q3 = ldg_stream16(base + (size_t)(r + 3 * RG) * nvec);
        eat(q0); eat(q1); eat(q2); eat(q3);
    }
    for (; r < r1; r += RG) eat(ldg_stream16(base + (size_t)r * nvec));
#pragma unroll
    for (int t = 0; t < 8; t++) s_col[(size_t)g * W + 8 * j + t] = cs[t];
    __syncthreads();
    unsigned long long tot = 0;
    for (int c = threadIdx.x; c < W; c += blockDim.x) {
        unsigned int sacc = 0;
        for (int k = 0; k < RG; k++) sacc += s_col[(size_t)k * W + c];
        atomicAdd(&colsum[(size_t)f * W + c], (unsigned long long)sacc);
        tot += sacc;
    }
    unsigned int mn = min(mn2 & 0xffffu, mn2 >> 16), mx = max(mx2 & 0xffffu, mx2 >> 16);
    mn = warp_min(mn); mx = warp_max(mx); tot = warp_sum(tot);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&acc[f].mn, mn);
        atomicMax(&acc[f].mx, mx);
        atomicAdd(&acc[f].sum, tot);
    }
}

// ------------------------------------------------------------------------------------------------ block helpers (fp64)
// image state: processed pixel = sign * v + off, with its current min / max
struct VmMap { int sign; long long off; long long mn, mx; };

__device__ inline void vm_ground(VmMap& m) { m.off -= m.mn; m.mx -= m.mn; m.mn = 0; }
__device__ inline void vm_invert(VmMap& m) {      // -a + max + min
    m.sign = -m.sign;
    m.off = -m.off + m.mx + m.mn;
}

// BaseImage.check_inversion(box_size=20, position=(0, 0)) (core/image.py:868-897) on the mapped image; `total` = sum of raw pixels.
// Block-wide: the 4 x 400 box pixels are spread over the threads (a single thread walking them was most of the kernel's time).
__device__ inline bool vm_check_inversion(const uint16_t* img, int H, int W, const VmMap& m, unsigned long long total, double* red) {
    // row_pos = col_pos = max(int(0 * N), 1) = 1; python slices [1:21] and [-21:-1], clipped like numpy
    const int bs = 20;
    auto clip = [](int v, int n) { return v < 0 ? max(v + n, 0) : min(v, n); };
    const int rr0[2] = {clip(1, H), clip(-1 - bs, H)}, rr1[2] = {clip(1 + bs, H), clip(-1, H)};
    const int cc0[2] = {clip(1, W), clip(-1 - bs, W)}, cc1[2] = {clip(1 + bs, W), clip(-1, W)};
    // np.mean((lt_upper, lt_lower, rt_upper, rt_lower)): the four boxes are stacked into one (4, 20, 20) array -> one mean over all
    // 1600 pixels (exact integer sum / count; sums of < 2^27 are exact in the fp64 block reduction)
    double s = 0, cnt = 0;
    for (int bi = 0; bi < 2; bi++)
        for (int bj = 0; bj < 2; bj++) {
            const int bh = rr1[bi] - rr0[bi], bw = cc1[bj] - cc0[bj];
            if (bh <= 0 || bw <= 0) continue;
            for (int i = threadIdx.x; i < bh * bw; i += blockDim.x) {
                const int r = rr0[bi] + i / bw, c = cc0[bj] + i % bw;
                s += (double)(m.sign * (long long)img[(size_t)r * W + c] + m.off);
                cnt += 1.0;
            }
        }
    s = blk_reduce<OpSum>(s, red);
    cnt = blk_reduce<OpSum>(cnt, red);
    const double avg = s / cnt;
    const long long tsum = m.sign * (long long)total + m.off * (long long)H * W;
    const double mean = (double)tsum / (double)((long long)H * W);
    return avg > mean;
}

struct VmProfOut { double center_idx, field_len, field_std; int status; };

struct VmWork {          // per-pair global work area
    double* vals;        // [W]
    PeakWork pw;
};

// Order statistics k and k2 (= k or k + 1) of n values that are all >= +0 (no NaN): 8-bit radix select on the IEEE bit patterns (8 passes of
// a 256-bin shared-memory histogram over the values that share the prefix found so far), then the successor: the same value when it
// occurs again, else the smallest larger value.  Results in red[34], red[35].  O(8 n) instead of the n^2 / threads of rank counting.
__device__ void vm_order_stat_pair(const double* v, int n, int k, int k2, double* red) {
    __shared__ unsigned s_hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_k, s_dup;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
    if (tid == 0) { s_prefix = 0; s_k = k; s_dup = 0; }
    for (int pass = 7; pass >= 0; pass--) {
        const int shift = pass * 8;
        for (int b = tid; b < 256; b += nt) s_hist[b] = 0;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        for (int j = tid; j < n; j += nt) {
            const unsigned long long key = (unsigned long long)__double_as_longlong(v[j]);
            if (pass == 7 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&s_hist[(unsigned)(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {
            unsigned c[8], t = 0;
#pragma unroll
            for (int e = 0; e < 8; e++) { c[e] = s_hist[lane * 8 + e]; t += c[e]; }
            unsigned inc = t;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
            const unsigned excl = inc - t;
            const unsigned kk = (unsigned)s_k;
            __syncwarp();
            if (kk >= excl && kk < inc) {
                unsigned acc = excl;
#pragma unroll
                for (int e = 0; e < 8; e++) {
                    if (kk >= acc && kk < acc + c[e]) {
                        s_prefix = prefix | ((unsigned long long)(lane * 8 + e) << shift);
                        s_k = (int)(kk - acc);
                        if (pass == 0) s_dup = (kk - acc + 1u < c[e]) ? 1 : 0;      // the value occurs again after rank k
                    }
                    acc += c[e];
                }
            }
        }
        __syncthreads();
    }
    const double sa = __longlong_as_double((long long)s_prefix);
    double sb = sa;
    if (k2 != k && !s_dup) {
        double m = VM_INF;
        for (int j = tid; j < n; j += nt) { const double x = v[j]; if (x > sa) m = fmin(m, x); }
        sb = blk_reduce<OpMin>(m, red);
    }
    __syncthreads();
    if (tid == 0) { red[34] = sa; red[35] = sb; }
}

// the profile of VMATLinearBase._roi_profiles for one image (vmat.py:766-783) + field_values() statistics (:741-742, 759)
__device__ void vm_roi_profile(const unsigned long long* colsum, int H, int W, const VmMap& m, VmWork& wk, double* red, VmProfOut* out) {
    double* v = wk.vals;
    const int tid = threadIdx.x, nt = blockDim.x;
    // np.mean(img.array, axis=0): exact integer column sum / H
    for (int j = tid; j < W; j += nt) {
        const long long t = m.sign * (long long)colsum[j] + m.off * (long long)H;
        v[j] = (double)t / (double)H;
    }
    __syncthreads();
    // FWXMProfile(ground=True, normalization=BEAM_CENTER)
    double mn = VM_INF;
    for (int j = tid; j < W; j += nt) mn = fmin(mn, v[j]);
    mn = blk_reduce<OpMin>(mn, red);
    for (int j = tid; j < W; j += nt) v[j] = v[j] - mn;
    __syncthreads();
    double l, r;
    int st = vm_edges(v, W, wk.pw, &l, &r);
    if (st) { if (tid == 0) { out->status = st; out->center_idx = NAN; out->field_len = 0; out->field_std = NAN; } __syncthreads(); return; }
    const double center = fabs(r - l) / 2 + l;          // cached_property: survives the later rescalings (core/profile.py:313-318)
    const double bcv = vm_lerp_at(v, W, center);
    __syncthreads();
    for (int j = tid; j < W; j += nt) v[j] = v[j] / bcv;
    __syncthreads();
    // profile.stretch(): ground(normalize(ground(v)) * (1 - 0), value=0)  (core/array_utils.py:142-168)
    mn = VM_INF;
    for (int j = tid; j < W; j += nt) mn = fmin(mn, v[j]);
    mn = blk_reduce<OpMin>(mn, red);
    double mx = -VM_INF;
    for (int j = tid; j < W; j += nt) { v[j] = v[j] - mn; mx = fmax(mx, v[j]); }
    mx = blk_reduce<OpMax>(mx, red);
    mn = VM_INF;
    for (int j = tid; j < W; j += nt) { v[j] = (v[j] / mx) * 1.0; mn = fmin(mn, v[j]); }
    mn = blk_reduce<OpMin>(mn, red);
    for (int j = tid; j < W; j += nt) v[j] = v[j] - mn + 0.0;
    __syncthreads();
    // np.percentile(values, 90): linear interpolation between the order statistics ip and ip + 1 (numpy _lerp).  The two order
    // statistics by rank counting (rank = number of samples that sort before this one, index as tie-break): W^2 / threads broadcast
    // reads of an L1-resident profile instead of a 66-pass block sort
    const double vi = (double)(W - 1) * (90.0 / 100.0);
    const double pf = floor(vi);
    const int ip = (int)pf, in = min(ip + 1, W - 1);
    const double g = vi - pf;
    // NaN anywhere (a flat / failed image): the rank-counting path below keeps its behaviour; otherwise every value is >= +0 after the
    // grounding above, IEEE bit patterns order like the values, and the two order statistics come from an 8-bit radix select
    int has_nan = 0;
    for (int j = tid; j < W; j += nt) has_nan |= (v[j] != v[j]) ? 1 : 0;
    has_nan = __syncthreads_or(has_nan);
    if (!has_nan) {
        vm_order_stat_pair(v, W, ip, in, red);
    } else {
        if (tid == 0) { red[34] = NAN; red[35] = NAN; }      // a profile with nan has no such ranks: numpy's percentile is nan as well
        __syncthreads();
        if (W <= 8 * nt) {
            // up to 8 samples per thread in registers, ONE pass over the profile (broadcast loads) ranks all of them
            double xi[8];
            int ii[8], rank[8];
    #pragma unroll
            for (int m = 0; m < 8; m++) { ii[m] = tid + m * nt; xi[m] = ii[m] < W ? v[ii[m]] : 0.0; rank[m] = 0; }
            for (int j = 0; j < W; j++) {
                const double xj = v[j];
    #pragma unroll
                for (int m = 0; m < 8; m++) rank[m] += (xj < xi[m] || (xj == xi[m] && j < ii[m])) ? 1 : 0;
            }
    #pragma unroll
            for (int m = 0; m < 8; m++) {
                if (ii[m] < W && rank[m] == ip) red[34] = xi[m];
                if (ii[m] < W && rank[m] == in) red[35] = xi[m];
            }
        } else {
            for (int i = tid; i < W; i += nt) {
                const double xi = v[i];
                int rank = 0;
                for (int j = 0; j < W; j++) { const double xj = v[j]; rank += (xj < xi || (xj == xi && j < i)) ? 1 : 0; }
                if (rank == ip) red[34] = xi;
                if (rank == in) red[35] = xi;
            }
        }
        __syncthreads();
    }
    __syncthreads();
    const double sa = red[34], sb = red[35];
    const double diff = sb - sa;
    double p90 = sa + diff * g;
    if (g >= 0.5) p90 = sb - diff * (1 - g);
    __syncthreads();
    for (int j = tid; j < W; j += nt) v[j] = v[j] / p90;
    __syncthreads();
    // field_values(in_field_ratio=0.8): fresh edges on the rescaled values (core/profile.py:295-311, 345-353)
    st = vm_edges(v, W, wk.pw, &l, &r);
    if (st) { if (tid == 0) { out->status = st; out->center_idx = center; out->field_len = 0; out->field_std = NAN; } __syncthreads(); return; }
    const double width = fmax(r, l) - fmin(r, l);
    const double f_left = l + (1 - 0.8) / 2 * width, f_right = r - (1 - 0.8) / 2 * width;
    const double lower = floor(fmin(f_left, f_right)), upper = ceil(fmax(f_left, f_right));
    const int lo = (int)fmax(lower, 0.0), hi = (int)fmin(upper, (double)(W - 1));
    const int len = hi >= lo ? hi - lo + 1 : 0;
    double s = 0;
    for (int j = lo + tid; j <= hi; j += nt) s += v[j];
    s = blk_reduce<OpSum>(s, red);
    const double mean = s / (double)len;
    double q = 0;
    for (int j = lo + tid; j <= hi; j += nt) { const double d = v[j] - mean; q += d * d; }
    q = blk_reduce<OpSum>(q, red);
    if (tid == 0) { out->status = 0; out->center_idx = center; out->field_len = (double)len; out->field_std = sqrt(q / (double)len); }
    __syncthreads();
}

struct VmPair {          // device-side per-pair state handed from k_vmat_profile to the segment kernel
    VmMap map[2];        // analysis maps of image 1 / 2 (after the constructor's ground / check_inversion)
    int open_idx;        // 0: image 1 is the open field
    int status;
    double x_fc;
};

__global__ void __launch_bounds__(VM_THREADS)
k_vmat_profile(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b, int n, int H, int W, epid_vmat_params p, const VmAcc* acc,
               const unsigned long long* colsum, char* work, size_t work_stride, int cap, int cap2, VmPair* pairs, epid_vmat_row* rows) {
    const int pi = blockIdx.x;
    __shared__ double red[40];
    __shared__ int s_small[VM_THREADS + 8];
    __shared__ VmProfOut pout[2];
    __shared__ VmMap smap[2];
    __shared__ int sinv[2];
    // carve the work area
    char* q = work + (size_t)pi * work_stride;
    auto take = [&](size_t bytes) { char* r = q; q += (bytes + 255) / 256 * 256; return r; };
    VmWork wk;
    wk.vals = (double*)take(sizeof(double) * W);
    wk.pw.cap = cap;
    wk.pw.prom = (double*)take(sizeof(double) * cap);
    wk.pw.width_height = (double*)take(sizeof(double) * cap);
    wk.pw.lip = (double*)take(sizeof(double) * cap);
    wk.pw.rip = (double*)take(sizeof(double) * cap);
    wk.pw.skey = (double*)take(sizeof(double) * cap2);
    wk.pw.idx = (int*)take(sizeof(int) * cap);
    wk.pw.lbase = (int*)take(sizeof(int) * cap);
    wk.pw.rbase = (int*)take(sizeof(int) * cap);
    wk.pw.flag = (int*)take(sizeof(int) * cap);
    wk.pw.sidx = (int*)take(sizeof(int) * cap2);
    wk.pw.s_small = s_small;

    for (int k = 0; k < 2; k++) {
        const int f = k == 0 ? pi : n + pi;
        const uint16_t* img = k == 0 ? a + (size_t)pi * H * W : b + (size_t)pi * H * W;
        VmMap m;      // every thread carries the same map (uniform decisions from block-wide reductions)
        m.sign = 1; m.off = 0; m.mn = acc[f].mn; m.mx = acc[f].mx;
        if (p.ground) vm_ground(m);                                               // _load_images (vmat.py:348-357)
        int inv = 0;
        if (p.check_inversion && vm_check_inversion(img, H, W, m, acc[f].sum, red)) { vm_invert(m); inv = 1; }   // vmat.py:721-725
        if (threadIdx.x == 0) { smap[k] = m; sinv[k] = inv; }
        __syncthreads();
        // _roi_profiles works on a deep copy: ground() and check_inversion() once more (vmat.py:771-773)
        VmMap c = m;
        vm_ground(c);
        if (vm_check_inversion(img, H, W, c, acc[f].sum, red)) vm_invert(c);
        vm_roi_profile(colsum + (size_t)f * W, H, W, c, wk, red, &pout[k]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        epid_vmat_row& R = rows[pi];
        memset(&R, 0, sizeof(R));
        VmPair& P = pairs[pi];
        P.map[0] = smap[0];
        P.map[1] = smap[1];
        R.inverted[0] = sinv[0];
        R.inverted[1] = sinv[1];
        R.nseg = p.nseg;
        for (int k = 0; k < 2; k++) { R.profile_center_idx[k] = pout[k].center_idx; R.field_len[k] = pout[k].field_len; R.field_std[k] = pout[k].field_std; }
        int status = pout[0].status ? pout[0].status : pout[1].status;
        // _identify_images (vmat.py:739-764)
        const double l1 = pout[0].field_len, l2 = pout[1].field_len;
        int open_idx;
        if (fabs(l1 - l2) > fmin(l1, l2)) open_idx = l1 > l2 ? 0 : 1;
        else if (pout[0].field_std > pout[1].field_std) open_idx = 1;      // image 1 is the DMLC image
        else open_idx = 0;
        if (p.invert_image_order) open_idx ^= 1;
        // _calculate_segments (vmat.py:814-828): round(open_prof.center_idx), image centre when outside the central third
        double x_fc = rint(pout[open_idx].center_idx);                    // python round(): half to even
        int warn = 0;
        const double iw = (double)W;
        if (!(iw / 3 <= x_fc && x_fc <= iw * 2 / 3)) { warn = 1; x_fc = rint(iw / 2 - 0.5); }
        P.open_idx = open_idx;
        P.status = status;
        P.x_fc = x_fc;
        R.status = status;
        R.open_is_first = open_idx == 0;
        R.center_warning = warn;
        R.x_field_center = x_fc;
    }
}

// ------------------------------------------------------------------------------------------------ segments
__global__ void __launch_bounds__(VM_THREADS)
k_vmat_segments(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b, int H, int W, epid_vmat_params p, const VmPair* pairs,
                epid_vmat_row* rows) {
    const int si = blockIdx.x, pi = blockIdx.y;
    __shared__ double red[40];
    const VmPair P = pairs[pi];
    const uint16_t* img[2] = {a + (size_t)pi * H * W, b + (size_t)pi * H * W};
    const uint16_t* io = img[P.open_idx];
    const uint16_t* id = img[P.open_idx ^ 1];
    const VmMap mo = P.map[P.open_idx], md = P.map[P.open_idx ^ 1];
    // Segment(Point(x, y), width = w_mm * dpmm, height = h_mm * dpmm) (vmat.py:829-841); y = open_image.center.y = H / 2 - 0.5
    const double cx = P.x_fc + p.offset_mm[si] * p.dpmm, cy = (double)H / 2 - 0.5;
    const double w = p.seg_w_mm * p.dpmm, h = p.seg_h_mm * p.dpmm;
    // Rectangle.vertices (rotation 0): TL, TR, BR, BL = centre -+ (w, h) / 2; pixels_flat's polygon (core/roi.py:647-656)
    const double tlx = -w / 2 + cx, tly = -h / 2 + cy, trx = w / 2 + cx, try_ = -h / 2 + cy;
    const double brx = w / 2 + cx, bry = h / 2 + cy, blx = -w / 2 + cx, bly = h / 2 + cy;
    const double vx[4] = {blx, brx - 1, trx - 1, tlx}, vy[4] = {bly - 1, bry - 1, try_, tly};
    const double xmin = fmin(fmin(vx[0], vx[1]), fmin(vx[2], vx[3])), xmax = fmax(fmax(vx[0], vx[1]), fmax(vx[2], vx[3]));
    const double ymin = fmin(fmin(vy[0], vy[1]), fmin(vy[2], vy[3])), ymax = fmax(fmax(vy[0], vy[1]), fmax(vy[2], vy[3]));
    const int r0 = (int)fmax(0.0, ymin), r1 = min((int)ceil(ymax), H - 1);
    const int c0 = (int)fmax(0.0, xmin), c1 = min((int)ceil(xmax), W - 1);
    const int bh = r1 - r0 + 1, bw = c1 - c0 + 1;
    double s = 0, cnt = 0;
    if (bh > 0 && bw > 0) {
        for (int i = threadIdx.x; i < bh * bw; i += blockDim.x) {
            const int r = r0 + i / bw, c = c0 + i % bw;
            if (!point_in_quad(vx, vy, (double)c, (double)r)) continue;
            const size_t o = (size_t)r * W + c;
            const double num = (double)(md.sign * (long long)id[o] + md.off), den = (double)(mo.sign * (long long)io[o] + mo.off);
            s += num / den;
            cnt += 1.0;
        }
    }
    s = blk_reduce<OpSum>(s, red);
    cnt = blk_reduce<OpSum>(cnt, red);
    const double mean = s / cnt;
    double q = 0;
    if (bh > 0 && bw > 0) {
        for (int i = threadIdx.x; i < bh * bw; i += blockDim.x) {
            const int r = r0 + i / bw, c = c0 + i % bw;
            if (!point_in_quad(vx, vy, (double)c, (double)r)) continue;
            const size_t o = (size_t)r * W + c;
            const double num = (double)(md.sign * (long long)id[o] + md.off), den = (double)(mo.sign * (long long)io[o] + mo.off);
            const double d = num / den - mean;
            q += d * d;
        }
    }
    q = blk_reduce<OpSum>(q, red);
    if (threadIdx.x == 0) {
        epid_vmat_row& R = rows[pi];
        R.r_corr[si] = mean * 100;
        R.stdev[si] = sqrt(q / cnt);
        R.center_x[si] = cx;
        R.center_y[si] = cy;
        R.npix[si] = cnt;
    }
}

__global__ void k_vmat_finalize(int n, epid_vmat_params p, epid_vmat_row* rows) {
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n) return;
    epid_vmat_row& R = rows[pi];
    const int ns = p.nseg;
    // _update_r_corrs (vmat.py:408-412), r_devs / avg_abs / avg / max (:419-436)
    double avg = 0;
    for (int i = 0; i < ns; i++) avg += R.r_corr[i];
    avg /= (double)ns;
    double sa = 0, sr = 0, mx = -VM_INF;
    bool any_nan = false;
    int all = 1;
    const double tol = p.tolerance_percent / 100;
    for (int i = 0; i < ns; i++) {
        const double d = ((R.r_corr[i] / avg) * 100) - 100;
        R.r_dev[i] = d;
        const int ok = fabs(d) < tol * 100;
        R.seg_passed[i] = ok;
        all &= ok;
        sa += fabs(d);
        sr += d;
        if (d != d) any_nan = true;
        mx = fmax(mx, fabs(d));
    }
    R.avg_abs_r_deviation = sa / (double)ns;
    R.avg_r_deviation = sr / (double)ns;
    R.max_r_deviation = any_nan ? NAN : mx;      // np.max propagates nan
    R.passed = all;
}

// ------------------------------------------------------------------------------------------------ ratio image
template <typename T>
__global__ void k_divide(const T* __restrict__ num, const T* __restrict__ den, double* __restrict__ out, size_t per, const double* so) {
    const int f = blockIdx.y;
    double sn = 1, on = 0, sd = 1, od = 0;
    if (so) { sn = so[4 * f]; on = so[4 * f + 1]; sd = so[4 * f + 2]; od = so[4 * f + 3]; }
    const T* pn = num + (size_t)f * per;
    const T* pd = den + (size_t)f * per;
    double* po = out + (size_t)f * per;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (size_t)gridDim.x * blockDim.x)
        po[i] = (sn * (double)pn[i] + on) / (sd * (double)pd[i] + od);
}

// ------------------------------------------------------------------------------------------------ DLG
constexpr int DLG_THREADS = 128;
constexpr int DLG_MAXLEN = 512;

__global__ void __launch_bounds__(DLG_THREADS)
k_dlg_leaf(const uint16_t* __restrict__ frames, int H, int W, int nleaf, const int* __restrict__ bottom, const int* __restrict__ top, int c0,
           int c1, double* measured, int* status) {
    const int li = blockIdx.x, fi = blockIdx.y;
    const uint16_t* img = frames + (size_t)fi * H * W;
    __shared__ double prof[DLG_MAXLEN];
    __shared__ double red[40];
    __shared__ double s_prom[DLG_MAXLEN / 2 + 1], s_wh[DLG_MAXLEN / 2 + 1], s_lip[DLG_MAXLEN / 2 + 1], s_rip[DLG_MAXLEN / 2 + 1], s_key[DLG_MAXLEN];
    __shared__ int s_idx[DLG_MAXLEN / 2 + 1], s_lb[DLG_MAXLEN / 2 + 1], s_rb[DLG_MAXLEN / 2 + 1], s_flag[DLG_MAXLEN / 2 + 1], s_sidx[DLG_MAXLEN];
    __shared__ int s_small[DLG_THREADS + 8];
    const int L = c1 - c0;
    const int rb = max(bottom[li], 0), rt = min(top[li], H);      // python slice [bottom:top] (both non-negative here)
    const int nr = rt - rb;
    double* out = measured + (size_t)fi * nleaf + li;
    if (nr <= 0 || L < 3) { if (threadIdx.x == 0) { *out = NAN; atomicMax(status, 2); } return; }
    // window.mean(axis=0): exact integer column sums / rows
    for (int j = threadIdx.x; j < L; j += DLG_THREADS) {
        unsigned long long s = 0;
        for (int r = rb; r < rt; r++) s += img[(size_t)r * W + c0 + j];
        prof[j] = (double)s / (double)nr;
    }
    __syncthreads();
    const double mid = prof[(int)((double)L / 2)];
    double s = 0;
    for (int j = threadIdx.x; j < L; j += DLG_THREADS) s += prof[j];
    s = blk_reduce<OpSum>(s, red);
    double mean = s / (double)L;
    if (mid < mean) {      // profile = invert(profile): -a + max + min
        double mn = VM_INF, mx = -VM_INF;
        for (int j = threadIdx.x; j < L; j += DLG_THREADS) { mn = fmin(mn, prof[j]); mx = fmax(mx, prof[j]); }
        mn = blk_reduce<OpMin>(mn, red);
        mx = blk_reduce<OpMax>(mx, red);
        for (int j = threadIdx.x; j < L; j += DLG_THREADS) prof[j] = -prof[j] + mx + mn;
        __syncthreads();
        s = 0;
        for (int j = threadIdx.x; j < L; j += DLG_THREADS) s += prof[j];
        s = blk_reduce<OpSum>(s, red);
        mean = s / (double)L;
    }
    PeakWork pw;
    pw.cap = L / 2 + 1;
    pw.idx = s_idx; pw.prom = s_prom; pw.lbase = s_lb; pw.rbase = s_rb; pw.width_height = s_wh; pw.lip = s_lip; pw.rip = s_rip;
    pw.flag = s_flag; pw.skey = s_key; pw.sidx = s_sidx; pw.s_small = s_small;
    PeakArgs a;
    a.hmin = -VM_INF; a.distance = 1; a.pmin = -1.0; a.wmin = 0.0; a.rel_height = 1.0 - 0.5; a.max_number = 1; a.sort_by_height = 0;
    const int c = block_find_peaks(prof, L, a, pw);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (c < 1) { *out = NAN; atomicMax(status, 2); }
        else *out = mid < mean ? -s_prom[0] : s_prom[0];      // the second test sees the (possibly inverted) profile's mean
    }
}

__global__ void k_dlg_fit(int n, int nleaf, const double* __restrict__ planned, const double* __restrict__ measured, double* slope,
                          double* intercept, double* dlg) {
    const int fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= n) return;
    const double* y = measured + (size_t)fi * nleaf;
    // scipy.stats.linregress: means, np.cov(x, y, bias=1) -> slope = ssxym / ssxm, intercept = ymean - slope * xmean
    double xm = 0, ym = 0;
    for (int i = 0; i < nleaf; i++) { xm += planned[i]; ym += y[i]; }
    xm /= (double)nleaf; ym /= (double)nleaf;
    double sxx = 0, sxy = 0;
    for (int i = 0; i < nleaf; i++) { const double dx = planned[i] - xm, dy = y[i] - ym; sxx += dx * dx; sxy += dx * dy; }
    sxx /= (double)nleaf; sxy /= (double)nleaf;
    const double sl = sxy / sxx, ic = ym - sl * xm;
    slope[fi] = sl;
    intercept[fi] = ic;
    dlg[fi] = ic / sl;
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_vmat_analyze(epid_ctx* ctx, const epid_batch* img1, const epid_batch* img2, const epid_vmat_params* p,
                                     epid_vmat_row* rows) {
    EPID_REQUIRE(ctx && img1 && img2 && p && rows, EPID_ERR_INVALID, "NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device"); return EPID_ERR_NO_DEVICE; }
    EPID_REQUIRE(img1->dtype == EPID_U16 && img2->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "VMAT analysis needs uint16 frames");
    EPID_REQUIRE(img1->n == img2->n && img1->h == img2->h && img1->w == img2->w, EPID_ERR_INVALID, "the two batches differ in shape");
    EPID_REQUIRE(p->nseg >= 1 && p->nseg <= EPID_VMAT_MAX_SEG, EPID_ERR_INVALID, "1..%d segments", EPID_VMAT_MAX_SEG);
    EPID_REQUIRE(p->dpmm > 0 && p->seg_w_mm > 0 && p->seg_h_mm > 0, EPID_ERR_INVALID, "bad geometry");
    EPID_REQUIRE(img1->w >= 8 && img1->h >= 42, EPID_ERR_INVALID, "frames too small");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = img1->n, H = img1->h, W = img1->w;
    const int cap = W / 2 + 1;
    int cap2 = 1;
    while (cap2 < W) cap2 <<= 1;
    auto rup = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t work_stride = rup(sizeof(double) * W) + 4 * rup(sizeof(double) * cap) + rup(sizeof(double) * cap2) + 4 * rup(sizeof(int) * cap) +
                               rup(sizeof(int) * cap2);
    const size_t b_acc = rup(sizeof(VmAcc) * 2 * n), b_col = rup(sizeof(unsigned long long) * 2 * (size_t)n * W);
    const size_t b_pairs = rup(sizeof(VmPair) * n), b_rows = rup(sizeof(epid_vmat_row) * n);
    int rc = ensure_scratch(ctx, b_acc + b_col + b_pairs + b_rows + work_stride * n + 1024);
    if (rc != EPID_OK) return rc;
    char* q = (char*)ctx->scratch;
    VmAcc* d_acc = (VmAcc*)q; q += b_acc;
    unsigned long long* d_col = (unsigned long long*)q; q += b_col;
    VmPair* d_pairs = (VmPair*)q; q += b_pairs;
    epid_vmat_row* d_rows = (epid_vmat_row*)q; q += b_rows;
    char* d_work = q;
    const uint16_t* a = (const uint16_t*)img1->dptr;
    const uint16_t* b = (const uint16_t*)img2->dptr;
    k_vmat_init<<<256, 256, 0, ctx->stream>>>(d_acc, d_col, (size_t)2 * n, (size_t)2 * n * W);
    const int nvec = W / 8;
    if ((W & 7) == 0 && nvec <= 1024 && (nvec & 31) == 0) {
        // warps must not straddle row groups for the final reductions to stay warp-uniform: nvec is a multiple of 32 here
        int RG = std::max(1, std::min(VM_ROWS / 4, 640 / nvec));
        while (nvec * RG > 1024) RG--;
        k_vmat_front_v16<<<dim3((H + VM_ROWS - 1) / VM_ROWS, 2 * n), nvec * RG, sizeof(unsigned int) * (size_t)RG * W, ctx->stream>>>(
            a, b, n, H, W, RG, d_acc, d_col);
    } else {
        int ft = ((W & 1) ? W : W / 2);
        ft = std::min(1024, (ft + 31) / 32 * 32);
        k_vmat_front<<<dim3((H + VM_ROWS - 1) / VM_ROWS, 2 * n), ft, 0, ctx->stream>>>(a, b, n, H, W, d_acc, d_col);
    }
    k_vmat_profile<<<n, VM_THREADS, 0, ctx->stream>>>(a, b, n, H, W, *p, d_acc, d_col, d_work, work_stride, cap, cap2, d_pairs, d_rows);
    k_vmat_segments<<<dim3(p->nseg, n), VM_THREADS, 0, ctx->stream>>>(a, b, H, W, *p, d_pairs, d_rows);
    k_vmat_finalize<<<(n + 127) / 128, 128, 0, ctx->stream>>>(n, *p, d_rows);
    ctx->launches += 5;
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaMemcpyAsync(rows, d_rows, sizeof(epid_vmat_row) * n, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    return EPID_OK;
}

extern "C" int32_t epid_divide(epid_ctx* ctx, const epid_batch* num, const epid_batch* den, const double* sign_off, epid_batch** out) {
    EPID_REQUIRE(ctx && num && den && out, EPID_ERR_INVALID, "NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device"); return EPID_ERR_NO_DEVICE; }
    EPID_REQUIRE(num->dtype == den->dtype && (num->dtype == EPID_U16 || num->dtype == EPID_F64), EPID_ERR_UNSUPPORTED,
                 "epid_divide: both uint16 or both float64");
    EPID_REQUIRE(num->n == den->n && num->h == den->h && num->w == den->w, EPID_ERR_INVALID, "the two batches differ in shape");
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = epid_batch_alloc(ctx, EPID_F64, num->n, num->h, num->w, out);
    if (rc != EPID_OK) return rc;
    double* d_so = nullptr;
    if (sign_off) {
        rc = ensure_scratch(ctx, sizeof(double) * 4 * num->n + 256);
        if (rc != EPID_OK) { epid_batch_free(*out); *out = nullptr; return rc; }
        d_so = (double*)ctx->scratch;
        EPID_CUDA(cudaMemcpyAsync(d_so, sign_off, sizeof(double) * 4 * num->n, cudaMemcpyHostToDevice, ctx->stream));
    }
    const size_t per = (size_t)num->h * num->w;
    const dim3 grid((unsigned)std::min<size_t>((per + 255) / 256, 1184), num->n);
    if (num->dtype == EPID_U16) k_divide<uint16_t><<<grid, 256, 0, ctx->stream>>>((const uint16_t*)num->dptr, (const uint16_t*)den->dptr, (double*)(*out)->dptr, per, d_so);
    else k_divide<double><<<grid, 256, 0, ctx->stream>>>((const double*)num->dptr, (const double*)den->dptr, (double*)(*out)->dptr, per, d_so);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    return EPID_OK;
}

extern "C" int32_t epid_dlg_analyze(epid_ctx* ctx, const epid_batch* b, int32_t nleaf, const int32_t* bottom, const int32_t* top, int32_t c0,
                                    int32_t c1, const double* planned, double* measured, double* slope, double* intercept, double* dlg) {
    EPID_REQUIRE(ctx && b && bottom && top && planned && measured && slope && intercept && dlg, EPID_ERR_INVALID, "NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device"); return EPID_ERR_NO_DEVICE; }
    EPID_REQUIRE(b->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "DLG analysis needs uint16 frames");
    EPID_REQUIRE(nleaf >= 2 && nleaf <= 1024, EPID_ERR_INVALID, "2..1024 leaves");
    EPID_REQUIRE(c0 >= 0 && c1 <= b->w && c1 - c0 >= 3 && c1 - c0 <= DLG_MAXLEN, EPID_ERR_INVALID, "profile window [%d, %d) unsupported", c0, c1);
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = b->n;
    auto rup = [](size_t v) { return (v + 255) / 256 * 256; };
    const size_t b_i = rup(sizeof(int) * nleaf), b_p = rup(sizeof(double) * nleaf), b_m = rup(sizeof(double) * (size_t)n * nleaf), b_o = rup(sizeof(double) * n);
    int rc = ensure_scratch(ctx, 2 * b_i + b_p + b_m + 3 * b_o + 512);
    if (rc != EPID_OK) return rc;
    char* q = (char*)ctx->scratch;
    int* d_bot = (int*)q; q += b_i;
    int* d_top = (int*)q; q += b_i;
    double* d_pl = (double*)q; q += b_p;
    double* d_me = (double*)q; q += b_m;
    double* d_sl = (double*)q; q += b_o;
    double* d_ic = (double*)q; q += b_o;
    double* d_dl = (double*)q; q += b_o;
    int* d_status = (int*)q;
    EPID_CUDA(cudaMemcpyAsync(d_bot, bottom, sizeof(int) * nleaf, cudaMemcpyHostToDevice, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(d_top, top, sizeof(int) * nleaf, cudaMemcpyHostToDevice, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(d_pl, planned, sizeof(double) * nleaf, cudaMemcpyHostToDevice, ctx->stream));
    EPID_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int), ctx->stream));
    k_dlg_leaf<<<dim3(nleaf, n), DLG_THREADS, 0, ctx->stream>>>((const uint16_t*)b->dptr, b->h, b->w, nleaf, d_bot, d_top, c0, c1, d_me, d_status);
    k_dlg_fit<<<(n + 63) / 64, 64, 0, ctx->stream>>>(n, nleaf, d_pl, d_me, d_sl, d_ic, d_dl);
    ctx->launches += 2;
    EPID_CUDA(cudaGetLastError());
    int hstatus = 0;
    EPID_CUDA(cudaMemcpyAsync(measured, d_me, sizeof(double) * (size_t)n * nleaf, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(slope, d_sl, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(intercept, d_ic, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(dlg, d_dl, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaMemcpyAsync(&hstatus, d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    EPID_REQUIRE(hstatus == 0, EPID_ERR_INVALID, "a leaf profile has no peak (the reference raises IndexError)");
    return EPID_OK;
}
